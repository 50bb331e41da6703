"""Where the time of a small validation call goes, and what the eight-lane field product costs against the per-thread one.

Default run: call time of kgv_validate_txs and kgv_validate_mempool_txs at 1 / 16 / 256 / 4 096 transactions (every entry
looked up in the table; host-pointer calls, each ends in a synchronisation; median of --reps after --warmup calls).

--profile DIR, a run of its own: torch.profiler around single kgv_validate_txs calls of 1 and 256 transactions, --reps
sessions each.  Per call (median over the sessions): the device time of the verify kernels, of every kernel and copy, and
the span from the first device activity to the last; the wall time of the call is the default run's.  Traces go to DIR.

Both print the card's name, power limit and SM clock, read in the same run, and one JSON line.

    python tools/prof_small_verify.py [--reps 30] [--warmup 5]
    python tools/prof_small_verify.py --profile /tmp/prof_small [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, Params, TransactionValidator  # noqa: E402
from rusty_kaspa_b200 import simgen  # noqa: E402
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else "unknown"


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def profile_call(fn, reps, trace):
    from torch.profiler import ProfilerActivity, profile
    rows = []
    for r in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        if r == 0:
            prof.export_chrome_trace(trace)
        ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
        kernels = {}
        for e in ev:
            k = e.name.split("<")[0].split("(")[0]
            kernels[k] = kernels.get(k, 0.0) + e.device_time / 1e3
        rows.append({"span_ms": (max(e.time_range.end for e in ev) - min(e.time_range.start for e in ev)) / 1e3,
                     "device_ms": sum(kernels.values()),
                     "verify_ms": sum(v for k, v in kernels.items() if "verify" in k),
                     "activities": len(ev), "kernels": kernels})
    med = {k: round(float(np.median([r[k] for r in rows])), 4) for k in ("span_ms", "device_ms", "verify_ms", "activities")}
    med["top"] = {k: round(v, 4) for k, v in sorted(rows[-1]["kernels"].items(), key=lambda kv: -kv[1])[:8]}
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    gpu = card()
    ctx = GpuContext(0)
    fk, fe, txs = simgen.funded_window(4096, n_keys=4096, n_nonces=4096, mix=(0.5, 0.2, 0.15, 0.15))
    us = GpuUtxoSet(ctx, 1 << 15)
    ae, ab = simgen.entries_to_arrays(fe)
    us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
    tv = TransactionValidator(ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    out = {"gpu": gpu, "sizes": {}}
    if a.profile:
        os.makedirs(a.profile, exist_ok=True)
        out["unit"] = "ms per kgv_validate_txs call, device activity from torch.profiler (median of sessions)"
        for n in (1, 256):
            b = build_batch(txs[:n])
            call = lambda: tv.validate_transactions_in_parallel(us, b, 10)
            for _ in range(a.warmup):
                call()
            out["sizes"][n] = profile_call(call, a.reps, os.path.join(a.profile, f"validate_txs_{n}.json"))
            print(n, "txs", json.dumps(out["sizes"][n]), flush=True)
    else:
        out["unit"] = "ms per call (median)"
        for n in (1, 16, 256, 4096):
            b = build_batch(txs[:n])
            t_old = median_ms(lambda: tv.validate_transactions_in_parallel(us, b, 10), a.reps, a.warmup)
            t_new = median_ms(lambda: tv.validate_mempool_transactions_in_utxo_context(us, b, 10), a.reps, a.warmup)
            out["sizes"][n] = {"kgv_validate_txs": round(t_old, 4), "kgv_validate_mempool_txs": round(t_new, 4)}
            print(f"{n:5d} txs  kgv_validate_txs {t_old:8.3f} ms   kgv_validate_mempool_txs {t_new:8.3f} ms", flush=True)
    print("card:", gpu)
    print(json.dumps(out))
    us.close()
    ctx.close()


if __name__ == "__main__":
    main()
