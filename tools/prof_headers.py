"""Throughput of kgv_hash_headers and kgv_validate_headers_in_isolation at 10^3, 10^5 and 10^6 headers, beside the C restatement
(tests/oracle_pow/ok_pow.c) on all host cores.

The headers are the 5 000 headers of the goref-notx-5000 fixture (5 to 10 levels, up to 8 parents per level), repeated with fresh nonces
and timestamps, so every header draws its own matrix.
  device ms   the call on device pointers (torch tensors) between two CUDA events on the context's stream, median of --reps calls
  wall ms     the call on host arrays (uploads, kernel, read-back, one synchronise), host clock, median of --reps calls
  oracle ms   ok_pow_validate_batch on os.cpu_count() threads, host clock, median of --oracle-reps runs (10^6 only with --oracle-1m)
The card's name, power limit and SM clock are printed with the numbers, read in the same run.

    python tools/prof_headers.py [--reps 5] [--out out/prof_headers.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batch(n, seed=1):
    import oracle_header as oh
    from rusty_kaspa_b200.headers import HeaderBatch
    _, hdrs = oh.fixture_headers(oh.FIXTURES[1])
    base = HeaderBatch.from_dicts(hdrs[1:])
    rng = np.random.default_rng(seed)
    h = np.resize(base.headers, n).copy()
    h["nonce"] = rng.integers(0, 2**63, n, dtype=np.uint64)
    h["timestamp"] += rng.integers(0, 1000, n, dtype=np.uint64)
    return HeaderBatch(h, base.level_len, base.parents)


def median_ms(f, reps):
    ts = []
    for _ in range(reps):
        ts.append(f())
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-reps", type=int, default=3)
    ap.add_argument("--oracle-1m", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import oracle_header as oh
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200.headers import HeaderRules, hash_headers, validate_headers_in_isolation
    ctx = rk.GpuContext(0)
    stream = torch.cuda.Stream()
    ctx.use_stream(stream.cuda_stream)
    lib = ctx._lib
    rules = HeaderRules(max_block_parents=81, max_block_level=254, timestamp_deviation_tolerance=600, now_ms=2**63)
    ok = oh.c_oracle()
    rows = []
    for n in (1000, 100_000, 1_000_000):
        b = batch(n)
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).cuda()
        dh, dp, dl = dev(b.headers), dev(b.parents), dev(b.level_len)
        dres, dhash, dpre = (torch.zeros(n * k, dtype=torch.uint8, device="cuda") for k in (24, 32, 32))
        torch.cuda.synchronize()

        def timed(call):
            def run():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                ctx._check(call())
                e1.record(stream)
                e1.synchronize()
                return e0.elapsed_time(e1)
            run()  # warm-up
            return median_ms(run, a.reps)

        hash_dev = timed(lambda: lib.kgv_hash_headers(ctx._h, dh.data_ptr(), n, dp.data_ptr(), len(b.parents), dl.data_ptr(), len(b.level_len),
                                                      dhash.data_ptr(), dpre.data_ptr()))
        val_dev = timed(lambda: lib.kgv_validate_headers_in_isolation(ctx._h, dh.data_ptr(), n, dp.data_ptr(), len(b.parents), dl.data_ptr(),
                                                                      len(b.level_len), ctypes.byref(rules), dres.data_ptr(), dhash.data_ptr(), None))

        def wall(f):
            def run():
                t = time.perf_counter()
                f()
                return 1e3 * (time.perf_counter() - t)
            run()
            return median_ms(run, a.reps)

        hash_wall = wall(lambda: hash_headers(ctx, b))
        val_wall = wall(lambda: validate_headers_in_isolation(ctx, b, rules, want_hash=True))
        # the GPU result equals the oracle's on the first 1 000 headers of each size
        want = oh.oracle_validate(ok, type(b)(b.headers[:1000], b.level_len, b.parents), rules)
        got = validate_headers_in_isolation(ctx, type(b)(b.headers[:1000], b.level_len, b.parents), rules, want_hash=True, want_pow=True)
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes()
        ora = None
        if n < 1_000_000 or a.oracle_1m:
            def orun():
                t = time.perf_counter()
                oh.oracle_validate(ok, b, rules)
                return 1e3 * (time.perf_counter() - t)
            ora = median_ms(orun, a.oracle_reps if n <= 1000 else 1)
        r = {"headers": n, "hash_device_ms": hash_dev, "hash_wall_ms": hash_wall, "validate_device_ms": val_dev, "validate_wall_ms": val_wall,
             "hash_headers_per_s": n / hash_dev * 1e3, "validate_headers_per_s": n / val_dev * 1e3, "oracle_ms": ora,
             "oracle_headers_per_s": (n / ora * 1e3) if ora else None, "oracle_threads": os.cpu_count()}
        rows.append(r)
        print(json.dumps(r), flush=True)
    info = card()  # after the runs: the SM clock under load
    print("card: %s" % info)
    print("%10s %12s %12s %14s %14s %14s %14s %14s" % ("headers", "hash dev ms", "hash wall ms", "hash hdr/s", "valid dev ms", "valid wall ms",
                                                         "valid hdr/s", "oracle hdr/s"))
    for r in rows:
        print("%10d %12.3f %12.3f %14.3e %14.3f %14.3f %14.3e %14s" % (r["headers"], r["hash_device_ms"], r["hash_wall_ms"], r["hash_headers_per_s"],
                                                                      r["validate_device_ms"], r["validate_wall_ms"], r["validate_headers_per_s"],
                                                                      "%.3e" % r["oracle_headers_per_s"] if r["oracle_headers_per_s"] else "not run"))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
