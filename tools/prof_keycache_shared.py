"""What sharing one device key cache between contexts (kgv_keycache_share) changes at the chain tip: a mempool context validates new
transactions (kgv_validate_mempool_txs), then a block context validates the same ones (kgv_validate_txs), both against one UTXO set.

Two arms, alternated call by call in one process, each on its own pair of contexts:
  separate   each context has its own cache: the keys the mempool met are cold for the block context
  shared     one cache, created on the block context and shared with the mempool context
Every call spends outputs of keys no earlier call used (a fresh slice of a funded window over 2^16 keys).  Reported per size (1, 16 and
256 transactions): median and p99 of the block context's kgv_validate_txs, its Schnorr and ECDSA hits per call (medians), and the device
memory the caches of each arm hold.  Verdicts are checked identical across the arms.  Prints the card's name, power limit and SM clock,
read in the same run, and one JSON line.

    python tools/prof_keycache_shared.py [--reps 100] [--warmup 5]
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

from prof_small_verify import card  # noqa: E402
from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, Params, TransactionValidator  # noqa: E402
from rusty_kaspa_b200 import simgen  # noqa: E402
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402
from rusty_kaspa_b200.validator import KeyCache  # noqa: E402

SIZES = (1, 16, 256)
CAP = (1 << 16, 1 << 14)  # Schnorr, ECDSA keys per cache


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


class Arm:
    def __init__(self, name, us, prm):
        self.name = name
        self.m, self.b = GpuContext(0), GpuContext(0)
        f0 = free_bytes()
        self.kb = KeyCache(self.b, *CAP)
        self.km = self.kb.on(self.m) if name == "shared" else KeyCache(self.m, *CAP)
        self.cache_bytes = f0 - free_bytes()
        self.us_m, self.us_b = us.on(self.m), us.on(self.b)
        self.tm, self.tb = TransactionValidator(self.m, prm), TransactionValidator(self.b, prm)
        self.t = {n: [] for n in SIZES}
        self.hits = {n: [] for n in SIZES}

    def hits_now(self):
        return self.kb.counters(False)["hits"], self.kb.counters(True)["hits"]

    def call(self, n, batch, timed):
        mres = self.tm.validate_mempool_transactions_in_utxo_context(self.us_m, batch, 10)[0]
        h0 = self.hits_now()
        t0 = time.perf_counter()
        res = self.tb.validate_transactions_in_parallel(self.us_b, batch, 10)
        t = (time.perf_counter() - t0) * 1e3
        h1 = self.hits_now()
        if timed:
            self.t[n].append(t)
            self.hits[n].append((h1[0] - h0[0], h1[1] - h0[1]))
        return mres["status"].tobytes() + res["status"].tobytes() + res["fee"].tobytes()

    def close(self):
        self.km.close()
        self.kb.close()
        self.m.close()
        self.b.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    gpu = card()
    rounds = a.warmup + a.reps
    per_round = sum(SIZES)
    fk, fe, txs = simgen.funded_window(rounds * per_round, seed=11, n_keys=1 << 16, n_nonces=1 << 12, mix=(0.6, 0.4, 0.0, 0.0))
    owner = GpuContext(0)
    us = GpuUtxoSet(owner, 1 << 17)
    ae, ab = simgen.entries_to_arrays(fe)
    us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
    prm = Params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    arms = [Arm("separate", us, prm), Arm("shared", us, prm)]
    nxt = 0
    for r in range(rounds):
        for n in SIZES:  # the same new transactions through both arms (their caches are apart): identical verdicts
            batch = build_batch(txs[nxt:nxt + n])
            nxt += n
            outs = [arm.call(n, batch, r >= a.warmup) for arm in (arms if r % 2 else arms[::-1])]
            assert outs[0] == outs[1], f"verdicts differ between the arms (round {r}, {n} transactions)"
    out = {"gpu": gpu, "unit": "ms per block-context kgv_validate_txs call", "reps": a.reps, "cache_keys": {"schnorr": CAP[0], "ecdsa": CAP[1]}}
    for arm in arms:
        out[arm.name] = {"cache_bytes_measured": int(arm.cache_bytes), "cache_bytes_records": int(sum(CAP) * (8320 + 44) * (2 if arm.name == "separate" else 1))}
        for n in SIZES:
            t = np.array(arm.t[n])
            h = np.array(arm.hits[n])
            out[arm.name][n] = {"median": round(float(np.median(t)), 4), "p99": round(float(np.percentile(t, 99)), 4),
                                "schnorr_hits": float(np.median(h[:, 0])), "ecdsa_hits": float(np.median(h[:, 1]))}
        print(arm.name, json.dumps(out[arm.name]), flush=True)
    for arm in arms:
        arm.close()
    us.close()
    owner.close()
    print("card:", gpu)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
