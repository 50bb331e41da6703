"""Call time of kgv_validate_mempool_txs against kgv_validate_txs on the same batch, every entry looked up in the table, at
1 / 16 / 256 / 4 096 transactions.  Host-pointer calls (each ends in a synchronisation), median of --reps after --warmup calls.
Prints the card's name and power limit, read in the same run, and one JSON line.

    python tools/prof_mempool.py [--reps 30] [--warmup 5]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    gpu = card()
    ctx = GpuContext(0)
    fk, fe, txs = simgen.funded_window(4096, n_keys=4096, n_nonces=4096, mix=(0.5, 0.2, 0.15, 0.15))
    us = GpuUtxoSet(ctx, 1 << 15)
    ae, ab = simgen.entries_to_arrays(fe)
    us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
    tv = TransactionValidator(ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    out = {"gpu": gpu, "unit": "ms per call (median)", "sizes": {}}
    for n in (1, 16, 256, 4096):
        b = build_batch(txs[:n])
        old = tv.validate_transactions_in_parallel(us, b, 10)
        new = tv.validate_mempool_transactions_in_utxo_context(us, b, 10)[0]
        assert (old["status"] == new["status"]).all() and (old["fee"] == new["fee"]).all()  # nothing differs on this batch
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
