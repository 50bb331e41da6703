#!/usr/bin/env python3
"""The per-launch key cache of the verify kernels (k_key_dedup + k_key_prepare, DESIGN.md §4 K1) at the bench shape and at its worst case.

    python tools/prof_key_cache.py [--n N] [--steps K] [--legs bench,distinct] [--profile DIR]

Legs (device-resident triples, L2 flushed before every timed call, CUDA events around each kgv_schnorr_verify call):
  bench     bench.py's workload: N triples over 65 536 keys (each key about 16 times)
  distinct  N triples drawn over N keys (about 0.64 N distinct): too many keys for records, so only the dedup pass is added
  sweep     N triples over N/64 ... N/2 distinct keys (a base set over about that many keys, tiled to N): where the comb records
            (at most N/COMB_USES keys) start to pay against the plain ones
Each leg prints one JSON line: ms per call (mean, min, max), verifies/s, the distinct keys, the keys used at least twice and the records a
launch makes and their form (every distinct key when there are at most n/2 and at most 2^17 of them, else none; comb records when there
are at most n/COMB_USES: key_form in kgv_lib.cu; counted from the keys on the host).
--profile DIR: a separate torch.profiler run of 3 calls per leg; the device time of every kernel and memset, summed per name, goes to
the JSON line (and the trace to DIR).  KGV_LIB selects the build of libkgv.so, so an older build can be timed the same way.
The generated triples are cached under the system's temporary directory (1 Mi distinct keys take a minute to generate).
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECORDS_MAX = 1 << 17
COMB_USES = 8  # KGV_COMB_USES in kgv_lib.cu
SWEEP = (64, 32, 16, 12, 10, 8, 6, 4, 3, 2)


def form(n, d):
    if d > min(n // 2, RECORDS_MAX):
        return "inline"
    return "comb" if COMB_USES * d <= n else "plain"


def triples(n, n_keys, seed):
    from rusty_kaspa_b200 import workload as W
    path = os.path.join(tempfile.gettempdir(), f"kgv_prof_key_cache_{n}_{n_keys}_{seed:x}.npz")
    if os.path.exists(path):
        z = np.load(path)
        return z["pk"], z["msg"], z["sig"], z["kind"]
    pk, msg, sig, kind = W.schnorr_triples(n, seed=seed, n_keys=n_keys, n_nonces=65536)
    np.savez(path, pk=pk, msg=msg, sig=sig, kind=kind)
    return pk, msg, sig, kind


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--legs", default="bench,distinct")
    ap.add_argument("--profile", metavar="DIR")
    args = ap.parse_args()
    import torch
    import rusty_kaspa_b200 as rk
    if not torch.cuda.is_available():
        raise SystemExit("prof_key_cache.py: no CUDA device")
    dev = torch.device("cuda", 0)
    ctx = rk.GpuContext(0)
    stream = torch.cuda.Stream(device=dev)
    ctx.use_stream(stream.cuda_stream)
    props = torch.cuda.get_device_properties(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    legs = []
    for leg in args.legs.split(","):
        legs += [(f"sweep_n/{u}", u) for u in SWEEP] if leg == "sweep" else [(leg, None)]
    for leg, u in legs:
        t0 = time.perf_counter()
        if u is None:
            n_keys = {"bench": 65536, "distinct": args.n}[leg]
            pk, msg, sig, kind = triples(args.n, n_keys, 0x6B61737061)
        else:  # a base set of 1.5 items per key over n_keys keys (about 0.78 n_keys distinct), tiled to n
            from rusty_kaspa_b200 import workload as W
            n_keys = int(args.n / u / 0.78)
            pk, msg, sig, kind = W.tile_triples(*triples(n_keys * 3 // 2, n_keys, 0x6B61737061), args.n)
        gen_s = time.perf_counter() - t0
        _, counts = np.unique(pk, axis=0, return_counts=True)
        repeated = int((counts >= 2).sum())
        with torch.cuda.stream(stream):
            dpk, dmsg, dsig = (torch.from_numpy(a).to(dev) for a in (pk, msg, sig))
            dst = torch.empty(args.n, dtype=torch.uint8, device=dev)
            call = lambda: ctx.verify_schnorr_batch(dpk, dmsg, dsig, n=args.n, status=dst)
            for _ in range(3):
                call()
            stream.synchronize()
            ms = []
            for _ in range(args.steps):
                flush.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                call()
                e1.record(stream)
                stream.synchronize()
                ms.append(e0.elapsed_time(e1))
            st = dst.cpu().numpy()
            assert int((st == 1).sum()) == int((kind == 0).sum()) and not (st[kind != 0] == 1).any()
            kernels = None
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                os.makedirs(args.profile, exist_ok=True)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        call()
                    stream.synchronize()
                prof.export_chrome_trace(os.path.join(args.profile, f"key_cache_{leg.replace('/', '_')}.json"))
                kernels = {}
                for ev in prof.events():
                    if ev.device_type.name == "CUDA":
                        k = ev.name.split("<")[0].split("(")[0]
                        kernels[k] = kernels.get(k, 0.0) + ev.device_time / 1e3 / 3
                kernels = {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}
        print(json.dumps({"leg": leg, "n": args.n, "n_keys": n_keys, "distinct_keys": int(len(counts)), "keys_used_twice_or_more": repeated,
                          "records_per_launch": len(counts) if len(counts) <= min(args.n // 2, RECORDS_MAX) else 0,
                          "form": form(args.n, len(counts)), "ms_mean": round(float(np.mean(ms)), 4), "ms_min": round(float(np.min(ms)), 4),
                          "ms_max": round(float(np.max(ms)), 4), "verifies_per_s": args.n / (float(np.mean(ms)) * 1e-3),
                          "kernel_ms_per_call": kernels, "lib": os.environ.get("KGV_LIB", "libkgv.so"), "gpu": props.name, "generation_s": round(gen_s, 1)}),
              flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
