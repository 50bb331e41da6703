"""Cost of the mempool's standardness policy.

1. Call time of kgv_validate_mempool_txs_with_policy (the default policy) against kgv_validate_mempool_txs_in_parallel on the same batches of
   1 / 16 / 256 / 4 096 transactions, every entry looked up in the table.  Host-pointer calls (each ends in a synchronisation), the two
   calls alternated, median of --reps after --warmup calls.
2. Device time of k_tx_standard_isolation and k_tx_standard_context (through kgv_check_txs_standard_in_isolation / _in_context) on
   device-resident batches of 10^6 transactions (2 inputs, 2 outputs each) and of 1 000 transactions of 1 000 inputs, every input and output
   standard (the kernels walk all of them), from torch.profiler: the mean kernel time over --reps calls.
Prints the card's name, power limit and current SM clock, read in the same run, and one JSON line.

    python tools/prof_standard.py [--reps 20] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, MempoolPolicy, Params, TransactionValidator  # noqa: E402
from rusty_kaspa_b200 import simgen  # noqa: E402
from rusty_kaspa_b200.txbatch import ENTRY_DTYPE, INPUT_DTYPE, OUTPUT_DTYPE, TX_DTYPE, build_batch  # noqa: E402
from rusty_kaspa_b200.validator import TX_MASSES_DTYPE  # noqa: E402

P2PK = bytes([0x20]) + bytes([1] * 32) + bytes([0xac])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else "unknown"


def median_ms(fns, reps, warmup):
    """alternates the calls of `fns`; the median host time of each"""
    for _ in range(warmup):
        for f in fns:
            f()
    t = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            t0 = time.perf_counter()
            f()
            t[k].append((time.perf_counter() - t0) * 1e3)
    return [float(np.median(x)) for x in t]


def synthetic(n_txs, n_in, n_out):
    """standard transactions: P2PK outputs of 10^8 sompi, 66-byte signature scripts, P2PK entries (numpy, no per-tx Python)"""
    T = np.zeros(n_txs, TX_DTYPE)
    I = np.zeros(n_txs * n_in, INPUT_DTYPE)
    O = np.zeros(n_txs * n_out, OUTPUT_DTYPE)
    E = np.zeros(n_txs * n_in, ENTRY_DTYPE)
    T["first_input"], T["n_inputs"] = np.arange(n_txs) * n_in, n_in
    T["first_output"], T["n_outputs"] = np.arange(n_txs) * n_out, n_out
    arena = np.zeros(256, np.uint8)
    arena[:34] = np.frombuffer(P2PK, np.uint8)
    I["sigscript_off"], I["sigscript_len"] = 64, 66
    O["value"], O["script_off"], O["script_len"] = 10**8, 0, 34
    E["amount"], E["script_off"], E["script_len"] = 10**9, 0, 34
    m = np.zeros(n_txs, TX_MASSES_DTYPE)
    m["compute_mass"], m["transient_mass"] = 3000, 3000
    return T, I, O, E, arena, m


def kernel_ms(ctx, T, I, O, E, arena, m, reps, warmup):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    t = {k: dev(v) for k, v in (("txs", T), ("inputs", I), ("outputs", O), ("entries", E), ("arena", arena), ("m", m),
                                ("sm", np.zeros(len(T), np.uint64)), ("fee", np.full(len(T), 10**6, np.uint64)))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(T), t["inputs"].data_ptr(), len(I), t["outputs"].data_ptr(), len(O), t["entries"].data_ptr(),
                     t["arena"].data_ptr(), len(arena))
    res = torch.zeros(len(T) * 16, dtype=torch.uint8, device="cuda")
    det = torch.zeros(len(T) * 8, dtype=torch.uint8, device="cuda")
    pol = MempoolPolicy()
    L = ctx._lib
    iso = lambda: ctx._check(L.kgv_check_txs_standard_in_isolation(ctx._h, ctypes.byref(cb), ctypes.byref(pol), t["m"].data_ptr(), res.data_ptr(), det.data_ptr()))
    con = lambda: ctx._check(L.kgv_check_txs_standard_in_context(ctx._h, ctypes.byref(cb), ctypes.byref(pol), t["m"].data_ptr(), t["sm"].data_ptr(),
                                                                  t["fee"].data_ptr(), res.data_ptr(), det.data_ptr()))
    out = {}
    for name, call in (("k_tx_standard_isolation", iso), ("k_tx_standard_context", con)):
        for _ in range(warmup):
            call()
        torch.cuda.synchronize()
        st = res.cpu().numpy().reshape(-1, 16)[:, 12]
        assert (st == 0).all(), np.unique(st)  # every rule walked to its end
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if name in e.key]
        assert ev and sum(e.count for e in ev) == reps, [e.key for e in prof.key_averages()]
        total_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
        out[name] = round(total_us / reps / 1000, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    gpu_before = card()
    ctx = GpuContext(0)
    fk, fe, txs = simgen.funded_window(4096, n_keys=4096, n_nonces=4096, mix=(0.5, 0.2, 0.15, 0.15))
    us = GpuUtxoSet(ctx, 1 << 15)
    ae, ab = simgen.entries_to_arrays(fe)
    us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
    tv = TransactionValidator(ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    pol = MempoolPolicy()
    out = {"gpu": gpu_before, "unit": "ms", "call": {}, "kernels": {}}
    for n in (1, 16, 256, 4096):
        b = build_batch(txs[:n])
        got = tv.validate_mempool_transactions_with_policy(us, b, 10, 10, pol)
        st = {int(s): int(c) for s, c in zip(*np.unique(got[0]["status"], return_counts=True))}
        t_old, t_new = median_ms([lambda: tv.validate_mempool_transactions_in_parallel_full(us, b, 10, 10),
                                  lambda: tv.validate_mempool_transactions_with_policy(us, b, 10, 10, pol)], a.reps, a.warmup)
        out["call"][n] = {"kgv_validate_mempool_txs_in_parallel": round(t_old, 4), "kgv_validate_mempool_txs_with_policy": round(t_new, 4), "statuses": st}
        print(f"{n:5d} txs  in_parallel {t_old:8.3f} ms   with_policy {t_new:8.3f} ms   statuses {st}", flush=True)
    for name, shape in (("1e6 txs x 2 inputs x 2 outputs", (10**6, 2, 2)), ("1000 txs x 1000 inputs", (1000, 1000, 2))):
        k = kernel_ms(ctx, *synthetic(*shape), a.reps, a.warmup)
        out["kernels"][name] = k
        print(f"{name}: {k}", flush=True)
    out["gpu_after"] = card()
    print("card (name, power limit, SM clock, max SM clock):", gpu_before, "/ after:", out["gpu_after"])
    print(json.dumps(out))
    us.close()
    ctx.close()


if __name__ == "__main__":
    main()
