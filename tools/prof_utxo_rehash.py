"""The UTXO table (K5) under churn, and what kgv_utxo_rehash gives back.  The bench's K5 shape: 4 Mi live entries (34-byte scripts) in a
2^24-slot (2 GiB) table, device-resident keys, CUDA events, warm-up, several repeats.

Reported at three points - freshly filled, after churn (erase 1 Mi live entries and insert 1 Mi new ones per call until fewer than 5 % of
the slots are EMPTY), after kgv_utxo_rehash at the same size:
  lookup rate of 4 Mi hits (every live key, new order every call) and of 4 Mi misses (fresh random keys), stats.longest_run, mean displacement.
Then the time of kgv_utxo_stats and kgv_utxo_rehash (whole calls, CUDA events) and of their kernels (torch.profiler, a separate run), with the
bytes each must move computed from the shapes, as a share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).

usage: python tools/prof_utxo_rehash.py [--log2-slots 24] [--live-log2 22] [--repeats 5] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import rusty_kaspa_b200 as rk
from rusty_kaspa_b200 import GpuUtxoSet
from rusty_kaspa_b200.txbatch import ENTRY_DTYPE

HBM_TBS = 3.35  # H100 SXM data sheet
SLOT, HEAD = 128, 64


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi(" + q + ")": out.splitlines()[0] if out else ""}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2-slots", type=int, default=24)
    ap.add_argument("--live-log2", type=int, default=22)
    ap.add_argument("--churn-log2", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this script measures on the GPU only")
    cap, n, m = 1 << a.log2_slots, 1 << a.live_log2, 1 << a.churn_log2
    dev = torch.device("cuda:0")
    ctx = rk.GpuContext(0)
    stream = torch.cuda.Stream(device=dev)
    ctx.use_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)  # the torch ops that make and shuffle keys run in the library's stream order
    lib, h = ctx._lib, ctx._h
    res = {"card": card(), "shape": {"capacity_slots": cap, "live": n, "churn_per_call": m, "script_len": 34}}
    print(json.dumps(res["card"]), flush=True)

    gen = torch.Generator(device=dev).manual_seed(7)
    rand_keys = lambda k: torch.randint(0, 256, (k, 36), dtype=torch.uint8, device=dev, generator=gen)
    rng = np.random.default_rng(7)
    ent = np.zeros(n, dtype=ENTRY_DTYPE)
    ent["amount"] = rng.integers(1, 1 << 40, size=n)
    ent["script_off"] = (np.arange(n, dtype=np.uint64) * 34 % (1 << 20)).astype(np.uint32)
    ent["script_len"] = 34
    arena = rng.integers(0, 256, size=(1 << 20) + 64, dtype=np.uint8)
    dent = torch.from_numpy(ent.view(np.uint8).reshape(-1, ENTRY_DTYPE.itemsize)).to(dev)
    darena = torch.from_numpy(arena).to(dev)
    live = rand_keys(n)  # live keys, device-resident (random 36-byte keys: distinct with overwhelming probability)
    us = GpuUtxoSet(ctx, cap)
    das = torch.empty(n, dtype=torch.uint8, device=dev)
    ctx._check(lib.kgv_utxo_apply_diff(h, us._h, None, 0, None, live.data_ptr(), dent.data_ptr(), darena.data_ptr(), len(arena), n, das.data_ptr()))
    stream.synchronize()
    assert us.count() == n

    de = torch.empty(n * ENTRY_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    df = torch.empty(n, dtype=torch.uint8, device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, reps=a.repeats):
        fn(); stream.synchronize()  # warm-up
        ts = []
        for _ in range(reps):
            ev0.record(stream); fn(); ev1.record(stream); stream.synchronize()
            ts.append(ev0.elapsed_time(ev1) * 1e-3)
        return float(np.median(ts)), float(min(ts)), float(max(ts))

    def lookups(keys):
        ctx._check(lib.kgv_utxo_lookup(h, us._h, keys.data_ptr(), n, de.data_ptr(), None, 0, df.data_ptr()))

    def point(name):
        s = us.stats()
        hits = live[torch.randperm(n, device=dev, generator=gen)].contiguous()
        misses = rand_keys(n)
        th = timed(lambda: lookups(hits))
        assert int(df.sum().item()) == n
        tm = timed(lambda: lookups(misses))
        assert int(df.sum().item()) == 0
        r = {"hit_lookups_per_s": n / th[0], "hit_ms_median_min_max": [t * 1e3 for t in th],
             "miss_lookups_per_s": n / tm[0], "miss_ms_median_min_max": [t * 1e3 for t in tm],
             "longest_run": s["longest_run"], "mean_displacement": s["sum_displacement"] / max(s["live"], 1), "max_displacement": s["max_displacement"],
             "empty_frac": s["empty"] / cap, "tombstone_frac": s["tombstones"] / cap, "live": s["live"], "rehashes": s["rehashes"]}
        res[name] = r
        print(name, json.dumps(r), flush=True)

    point("fresh")
    # churn: erase m live entries, insert m new ones, until EMPTY < 5 % of the slots
    drs = torch.empty(m, dtype=torch.uint8, device=dev)
    calls, t0 = 0, time.perf_counter()
    while True:
        sel = torch.randperm(n, device=dev, generator=gen)[:m]
        old, new = live[sel].contiguous(), rand_keys(m)
        ctx._check(lib.kgv_utxo_apply_diff(h, us._h, old.data_ptr(), m, drs.data_ptr(), new.data_ptr(), dent.data_ptr(), darena.data_ptr(), len(arena), m, das.data_ptr()))
        live[sel] = new
        calls += 1
        if calls % 4 == 0:
            s = us.stats()
            assert s["insert_failures"] == 0 and s["live"] == n
            if s["empty"] < cap // 20:
                break
    stream.synchronize()
    res["churn"] = {"calls": calls, "erased_and_inserted": calls * m, "per_capacity": calls * m / cap, "seconds": time.perf_counter() - t0}
    print("churn", json.dumps(res["churn"]), flush=True)
    point("churned")
    digest = us.digest()

    # whole calls, CUDA events on the context's stream; kgv_utxo_rehash synchronises inside (after its stats pass) and allocates
    t_stats = timed(lambda: us.stats())
    ts = []
    for r in range(a.repeats + 1):  # the first is the warm-up
        ev0.record(stream); us.rehash(); ev1.record(stream); stream.synchronize()
        ts.append(ev0.elapsed_time(ev1) * 1e-3)
        ctx.synchronize()  # releases the previous arrays the rehash parked (outside the timed window)
    t_rehash = (float(np.median(ts[1:])), float(min(ts[1:])), float(max(ts[1:])))
    res["rehash_call_ms_median_min_max"] = [t * 1e3 for t in t_rehash]
    res["stats_call_ms_median_min_max"] = [t * 1e3 for t in t_stats]
    assert us.digest() == digest and us.count() == n
    point("rehashed")

    # kernel times, separate profiled run
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.repeats):
            us.stats()
            us.rehash()
            ctx.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.key.startswith(("k_utxo_stats", "k_utxo_rehash", "_Z12k_utxo_stats", "_Z13k_utxo_rehash", "_Z17k_utxo_stats_join")) or "Memset" in e.key:
            us_dev = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            kern[e.key] = {"calls": e.count, "mean_us": us_dev / max(e.count, 1)}
    res["kernels"] = kern
    print("kernels", json.dumps(kern), flush=True)

    # bytes from the shapes
    b_stats = cap * HEAD
    b_rehash_kernel = cap * HEAD + n * (SLOT - HEAD) + n * SLOT
    b_clear = cap * SLOT
    b_rehash_call = b_stats + b_rehash_kernel + b_clear  # the call's own stats pass (arena sizing) + clear of the new array + the move
    peak = HBM_TBS * 1e12

    def share(b, t):
        return {"bytes": b, "seconds": t, "GB_per_s": b / t * 1e-9, "share_of_3.35TBps_datasheet": b / t / peak}

    res["stats_call"] = share(b_stats, t_stats[0])
    res["rehash_call"] = share(b_rehash_call, t_rehash[0])
    # kernel shares where the profiler names the kernels
    for key, v in kern.items():
        if "k_utxo_rehash" in key:
            res["rehash_kernel"] = share(b_rehash_kernel, v["mean_us"] * 1e-6)
        elif "k_utxo_stats" in key and "join" not in key:
            res["stats_kernel"] = share(b_stats, v["mean_us"] * 1e-6)
    res["bytes_note"] = ("stats: every slot head (64 B) read.  rehash kernel: every head read, the other 64 B of every live slot read, every live slot "
                         "written (128 B).  rehash call: + its stats pass + the new array cleared (128 B per slot).  Shares are of the H100 SXM "
                         "data-sheet HBM bandwidth, 3.35 TB/s, not of a measured peak.")
    for k in ("stats_call", "rehash_call", "stats_kernel", "rehash_kernel"):
        if k in res:
            print(k, json.dumps(res[k]), flush=True)
    us.close(); ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_utxo_rehash.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
