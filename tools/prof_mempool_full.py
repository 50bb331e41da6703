"""Cost of the isolation and finality stage.

1. Call time of kgv_validate_mempool_txs_in_parallel (isolation -> finality -> UTXO context) against kgv_validate_mempool_txs (UTXO
   context only) on the same batches of 1 / 16 / 256 / 4 096 transactions, every entry looked up in the table.  Host-pointer calls (each
   ends in a synchronisation), the two calls alternated, median of --reps after --warmup calls.
2. kgv_validate_txs_in_isolation alone on a device-resident batch of 10^6 transactions (2 inputs, 2 outputs each), and on 1 000
   transactions of 1 000 inputs (the sorted duplicate check): CUDA events around --reps calls.
Prints the card's name, power limit and maximum SM clock, read in the same run, and one JSON line.

    python tools/prof_mempool_full.py [--reps 30] [--warmup 5]
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

from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, Params, TransactionValidator, TxRules  # noqa: E402
from rusty_kaspa_b200 import simgen  # noqa: E402
from rusty_kaspa_b200.txbatch import INPUT_DTYPE, OUTPUT_DTYPE, TX_DTYPE, build_batch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
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


def synthetic(n_txs, n_in, n_out, seed=1):
    """a batch of valid native transactions with distinct random outpoints (numpy, no per-tx Python)"""
    rng = np.random.default_rng(seed)
    T = np.zeros(n_txs, TX_DTYPE)
    I = np.zeros(n_txs * n_in, INPUT_DTYPE)
    O = np.zeros(n_txs * n_out, OUTPUT_DTYPE)
    T["first_input"] = np.arange(n_txs) * n_in
    T["n_inputs"] = n_in
    T["first_output"] = np.arange(n_txs) * n_out
    T["n_outputs"] = n_out
    I["prev_txid"] = rng.integers(0, 256, (len(I), 32), dtype=np.uint8)
    I["prev_index"] = rng.integers(0, 2**32, len(I), dtype=np.uint64).astype(np.uint32)
    I["sigscript_len"] = 66
    I["sig_op_count"] = 1
    I["sequence"] = 2**64 - 1
    O["value"] = rng.integers(1, 10**12, len(O), dtype=np.uint64)
    O["script_len"] = 34
    arena = np.zeros(256, np.uint8)
    return T, I, O, arena


def isolation_device_ms(ctx, T, I, O, arena, reps, warmup):
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    t = {k: dev(v) for k, v in (("txs", T), ("inputs", I), ("outputs", O), ("arena", arena))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(T), t["inputs"].data_ptr(), len(I), t["outputs"].data_ptr(), len(O), None, t["arena"].data_ptr(), len(arena))
    res = torch.zeros(len(T) * 16, dtype=torch.uint8, device="cuda")
    ms = torch.zeros(len(T) * 16, dtype=torch.uint8, device="cuda")
    rules = TxRules()
    stream = torch.cuda.current_stream()
    ctx._check(ctx._lib.kgv_set_stream(ctx._h, ctypes.c_void_p(stream.cuda_stream)))
    call = lambda: ctx._check(ctx._lib.kgv_validate_txs_in_isolation(ctx._h, ctypes.byref(cb), ctypes.byref(rules), 10, 10, 0, res.data_ptr(), ms.data_ptr()))
    for _ in range(warmup):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ctx._check(ctx._lib.kgv_reset_stream(ctx._h))
    st = res.cpu().numpy().view(np.uint8).reshape(-1, 16)[:, 12]
    assert (st == 0).all(), np.unique(st)
    return e0.elapsed_time(e1) / reps


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
    out = {"gpu": gpu, "unit": "ms (median per call)", "mempool": {}, "isolation": {}}
    for n in (1, 16, 256, 4096):
        b = build_batch(txs[:n])
        old = tv.validate_mempool_transactions_in_utxo_context(us, b, 10)
        new = tv.validate_mempool_transactions_in_parallel_full(us, b, 10, 10)
        assert (old[0] == new[0]).all() and (old[1] == new[1]).all()  # every transaction passes isolation and finality here
        t_old, t_new = median_ms([lambda: tv.validate_mempool_transactions_in_utxo_context(us, b, 10),
                                  lambda: tv.validate_mempool_transactions_in_parallel_full(us, b, 10, 10)], a.reps, a.warmup)
        out["mempool"][n] = {"kgv_validate_mempool_txs": round(t_old, 4), "kgv_validate_mempool_txs_in_parallel": round(t_new, 4)}
        print(f"{n:5d} txs  kgv_validate_mempool_txs {t_old:8.3f} ms   kgv_validate_mempool_txs_in_parallel {t_new:8.3f} ms", flush=True)
    for name, shape in (("1e6 txs x 2 inputs", (10**6, 2, 2)), ("1000 txs x 1000 inputs", (1000, 1000, 2))):
        ms = isolation_device_ms(ctx, *synthetic(*shape), a.reps, a.warmup)
        out["isolation"][name] = round(ms, 4)
        print(f"kgv_validate_txs_in_isolation, {name}: {ms:.3f} ms", flush=True)
    print("card:", gpu)
    print(json.dumps(out))
    us.close()
    ctx.close()


if __name__ == "__main__":
    main()
