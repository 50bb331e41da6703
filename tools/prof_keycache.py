"""What the device key cache (kgv_keycache) changes: call times with the cache off, cold (emptied before each call: every key a miss, stored
by the call) and warm (every key stored), the arms alternated call by call in one process, verdicts checked byte-identical across arms.

Default run (medians of --reps calls after --warmup):
  small    kgv_validate_txs and kgv_validate_mempool_txs on bench.py's small_batches shape (1, 16 and 256 transactions, host arrays);
           warm_after_cold is the call right after a cold one (it waits for that call's deferred insert), warm follows an untimed warm call
  large    kgv_schnorr_verify on device arrays: 1 Mi triples over 65 536 keys, one e2e chunk (202 752 triples) at about 3 uses per key,
           1 Mi triples over 1 Mi keys
  replay   one kgv_replay_window of a generated chain (off and warm)
--profile DIR, a run of its own: torch.profiler around single kgv_validate_txs calls of 1 and 256 transactions, off and warm: the verify
kernels' device time (median of --reps sessions), traces to DIR.

Both print the card's name, power limit and SM clock, read in the same run, and one JSON line.

    python tools/prof_keycache.py [--reps 30] [--warmup 5]
    python tools/prof_keycache.py --profile /tmp/prof_keycache [--reps 10]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from prof_small_verify import card, profile_call  # noqa: E402
from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, Params, TransactionValidator  # noqa: E402
from rusty_kaspa_b200 import simgen, workload as W  # noqa: E402
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402
from rusty_kaspa_b200.validator import KeyCache  # noqa: E402


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def arms(kc, call, reps, warmup, arm_names=("off", "cold", "warm_after_cold", "warm"), sync=None):
    """median ms per arm, the arms alternated; every arm's output must equal the first one's"""
    ts = {a: [] for a in arm_names}
    ref = None
    for r in range(warmup + reps):
        for a in arm_names:
            if a == "off":
                kc.detach()
            else:
                kc.attach()
                if a == "cold":
                    kc.clear()
            if a == "warm":
                call()
            if sync:
                sync()
            t, out = timed(call)
            key = out if isinstance(out, bytes) else np.asarray(out).tobytes()
            if ref is None:
                ref = key
            assert key == ref, f"arm {a}: output differs from the first call's"
            if r >= warmup:
                ts[a].append(t)
    kc.attach()
    return {a: round(float(np.median(v)), 4) for a, v in ts.items()}


def small(ctx, kc, reps, warmup):
    fk, fe, txs = simgen.funded_window(256, n_keys=64, n_nonces=64)
    ae, ab = simgen.entries_to_arrays(fe)
    us = GpuUtxoSet(ctx, 4096)
    us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
    tv = TransactionValidator(ctx, Params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    out = {}
    for n in (1, 16, 256):
        b = build_batch(txs[:n])
        v = lambda: tv.validate_transactions_in_parallel(us, b, 10)["status"].copy()
        m = lambda: tv.validate_mempool_transactions_in_utxo_context(us, b, 10)[0]["status"].copy()
        out[n] = {"kgv_validate_txs": arms(kc, v, reps, warmup), "kgv_validate_mempool_txs": arms(kc, m, reps, warmup)}
        print(n, "txs", json.dumps(out[n]), flush=True)
    us.close()
    return out, tv, us


def large(ctx, kc, reps, warmup):
    import torch
    out = {}
    for name, n, n_keys in (("1Mi_over_64Ki_keys", 1 << 20, 1 << 16), ("e2e_chunk_3_uses", 202_752, 67_584), ("1Mi_over_1Mi_keys", 1 << 20, 1 << 20)):
        pk, msg, sig, _ = W.schnorr_triples(n, seed=17, n_keys=n_keys, n_nonces=4096, frac_bitflip=0.01, frac_adversarial=0.01)
        d = [torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda() for a in (pk, msg, sig)]
        st = torch.empty(n, dtype=torch.uint8, device="cuda")

        def call():
            ctx.verify_schnorr_batch(*d, n=n, status=st)
            torch.cuda.synchronize()
            return st.cpu().numpy()
        out[name] = arms(kc, call, reps, warmup, sync=torch.cuda.synchronize)
        out[name]["counters"] = kc.counters(False)
        print(name, json.dumps(out[name]), flush=True)
        del d, st
    return out


def replay(ctx, kc, reps, warmup):
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_BLOCK_DTYPE
    g = simgen.FastDag(seed=5, n_keys=1024, n_nonces=4096, coinbase_maturity=3, frac_invalid=0.01, coinbase_outputs=64)
    g.generate(100, 100)
    b, first, pov = g.take()
    arr = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
    arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1

    def fresh():  # the window from an empty UTXO set, timed alone
        r = DagReplayer(ctx, Params(coinbase_maturity=3, storage_mass_parameter=g.C), 1 << 16)
        t, (got, acc) = timed(lambda: r.replay_window(b, arr, want_accept=True))
        d = r.us.digest()
        r.close()
        return t, got["status"].tobytes() + acc.tobytes() + d
    ts = {"off": [], "warm": []}
    ref = None
    for r in range(warmup + reps):
        for a in ("off", "warm"):
            (kc.detach if a == "off" else kc.attach)()
            t, key = fresh()
            ref = ref or key
            assert key == ref, f"replay arm {a} differs"
            if r >= warmup:
                ts[a].append(t)
    kc.attach()
    g.close()
    out = {"n_txs": int(len(b.txs)), **{a: round(float(np.median(v)), 3) for a, v in ts.items()}}
    print("replay", json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", default=None)
    ap.add_argument("--small-only", action="store_true", help="the small-call arms alone")
    ap.add_argument("--large-only", action="store_true", help="the large-launch arms alone")
    a = ap.parse_args()
    gpu = card()
    ctx = GpuContext(0)
    kc = KeyCache(ctx, 1 << 18, 1 << 14)
    out = {"gpu": gpu, "unit": "ms per call (median)"}
    if a.profile:
        os.makedirs(a.profile, exist_ok=True)
        fk, fe, txs = simgen.funded_window(256, n_keys=64, n_nonces=64)
        ae, ab = simgen.entries_to_arrays(fe)
        us = GpuUtxoSet(ctx, 4096)
        us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
        tv = TransactionValidator(ctx, Params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
        out["unit"] = "ms per kgv_validate_txs call, device activity from torch.profiler (median of sessions)"
        out["profile"] = {}
        for n in (1, 256):
            b = build_batch(txs[:n])
            call = lambda: tv.validate_transactions_in_parallel(us, b, 10)
            for arm in ("off", "warm"):
                (kc.detach if arm == "off" else kc.attach)()
                for _ in range(a.warmup):
                    call()
                out["profile"][f"{n}_{arm}"] = profile_call(call, a.reps, os.path.join(a.profile, f"validate_txs_{n}_{arm}.json"))
                print(n, arm, json.dumps(out["profile"][f"{n}_{arm}"]), flush=True)
        us.close()
    else:
        if not a.large_only:
            out["small"], _, _ = small(ctx, kc, a.reps, a.warmup)
        if a.large_only:
            out["large"] = large(ctx, kc, a.reps, a.warmup)
        elif not a.small_only:
            out["large"] = large(ctx, kc, a.reps, a.warmup)
            out["replay"] = replay(ctx, kc, a.reps, a.warmup)
    print("card:", gpu)
    print(json.dumps(out))
    kc.close()
    ctx.close()


if __name__ == "__main__":
    main()
