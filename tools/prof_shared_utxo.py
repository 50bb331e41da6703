"""Mempool calls against a UTXO set that block processing replays into and commits, in one process (include/kgv.h, Threading).

Mempool batches of 1, 16 and 256 transactions (bench.py's small_batches shape: 1-/2-input P2PK Schnorr, host arrays) are validated with
kgv_validate_mempool_txs against the committed set; their funding outputs are in it.  Host-timed to completion, median and p99 per size:
  alone         no other work on the device
  same_context  issued on the context that replays (from another thread): the only safe form before tables could be shared; each call waits
                behind the context's mutex for the replay call in flight
  shared        from a second context, while the first replays config-3-shaped windows (FastDag, 150 transactions per block, --window
                blocks per kgv_replay_window) into a view over the set and commits each (kgv_utxo_view_commit)
  shared_hp     as shared, the second context on a high-priority stream (kgv_set_stream)
and the replay throughput (transactions of the windows per second of the replay-and-commit loop) without and with that mempool load.  The
writer loops over the windows (Setup) until the mempool side has made --calls calls of each size, at most --max-passes passes; each
loaded case reports its calls and passes.

Prints the card's name, power limit and SM clock, read in the same run, and one JSON line.

    python tools/prof_shared_utxo.py [--window 1024] [--windows 12] [--calls 200] [--max-passes 40]
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from prof_small_verify import card  # noqa: E402
from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, Params, TransactionValidator, simgen  # noqa: E402
from rusty_kaspa_b200.replay import REPLAY_BLOCK_DTYPE, DagReplayer  # noqa: E402
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402
from rusty_kaspa_b200.validator import RESULT_DTYPE  # noqa: E402
from rusty_kaspa_b200.verifier import _c_batch  # noqa: E402

SIZES = (1, 16, 256)


def chain(window, n_windows):
    gen = simgen.FastDag(seed=0x6B61737061, n_keys=1024, n_nonces=4096, frac_two_inputs=0.5, frac_invalid=0.01, coinbase_outputs=16)
    wins = []
    for _ in range(n_windows):
        gen.generate(window, 150)
        b, first, pov = gen.take()
        arr = np.zeros(window, dtype=REPLAY_BLOCK_DTYPE)
        arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1
        wins.append((b, arr))
    return wins, Params(coinbase_maturity=gen.maturity, storage_mass_parameter=gen.C)


class Setup:
    """A fresh committed set on ctx_a (the mempool funding outputs loaded), a view over it, and the replay-and-commit loop.  One pass
    replays and commits every window; the next pass first undoes the previous one (each window's UtxoDiff, taken with kgv_replay_diffs in
    the warm-up pass and the same in every pass, applied reversed with kgv_utxo_apply_diff, then a same-size kgv_utxo_rehash to drop the
    tombstones), so the loop can run as long as the mempool side needs.  Throughput counts the forward passes only."""

    def __init__(self, ctx_a, wins, prm, fund):
        self.ctx, self.wins, self.prm = ctx_a, wins, prm
        self.base = GpuUtxoSet(ctx_a, 1 << 24)
        self.base.apply_diff(add_keys36=fund[0], add_entries=fund[1], add_bytes=fund[2])
        self.view = self.base.compose(1 << 22)
        self.done, self.enough = threading.Event(), threading.Event()
        self.statuses = []

    def loop(self, max_passes=1, diffs=None):
        """diffs: None (one pass, and self.diffs = every window's UtxoDiff), or those of an earlier run to undo passes with"""
        lib, h = self.ctx._lib, self.ctx._h
        fwd_s, n = 0.0, 0
        self.diffs = []
        for p in range(max_passes if diffs else 1):
            if p:
                for d in reversed(diffs):
                    d.apply(self.base, 0, reverse=True)
                self.base.rehash(0)
            t0 = time.perf_counter()
            for b, arr in self.wins:
                cb = _c_batch(b, with_entries=False)
                res = np.zeros(len(b.txs), dtype=RESULT_DTYPE)
                self.ctx._check(lib.kgv_replay_window(h, self.view._h, C.byref(cb), arr.ctypes.data, len(arr), C.byref(self.prm), res.ctypes.data, None, None))
                if diffs is None:
                    self.diffs.append(DagReplayer.replay_diffs(self, [0, len(arr)]))
                self.view.commit()
                if p == 0:
                    self.statuses.append(res["status"].copy())
                n += len(b.txs)
            self.ctx.synchronize()
            fwd_s += time.perf_counter() - t0
            if self.enough.is_set():
                break
        self.passes = p + 1
        self.tx_per_s = n / fwd_s
        self.done.set()

    def close(self):
        self.view.close()
        self.base.close()


def mempool_calls(tv, us, batches, vdaa, calls, stop=None):
    """round robin over the sizes until each has `calls` calls (or `stop` is set); ms per call per size"""
    ts = {n: [] for n in SIZES}
    while min(len(v) for v in ts.values()) < calls and not (stop is not None and stop.done.is_set()):
        for n in SIZES:
            t0 = time.perf_counter()
            res = tv.validate_mempool_transactions_in_utxo_context(us, batches[n], vdaa)[0]
            ts[n].append((time.perf_counter() - t0) * 1e3)
            assert (res["status"] == 0).all(), "a funded mempool transaction was rejected"
    if stop is not None:
        stop.enough.set()
    return ts


def summary(ts):
    return {str(n): {"calls": len(v), "median_ms": round(float(np.median(v)), 4) if v else None,
                     "p99_ms": round(float(np.percentile(v, 99)), 4) if v else None} for n, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=int, default=1024)
    ap.add_argument("--windows", type=int, default=12)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--max-passes", type=int, default=40)
    a = ap.parse_args()
    import torch
    info = card()
    wins, prm = chain(a.window, a.windows)
    fk, fe, txs = simgen.funded_window(256, n_keys=64, n_nonces=64)
    ae, ab = simgen.entries_to_arrays(fe)
    fund = (fk, ae, ab)
    batches = {n: build_batch(txs[:n]) for n in SIZES}
    vdaa = 1000
    ctx_a, ctx_b = GpuContext(0), GpuContext(0)
    tv_a, tv_b = TransactionValidator(ctx_a, prm), TransactionValidator(ctx_b, prm)
    out = {"card": info, "window_blocks": a.window, "windows": a.windows, "window_txs": int(np.mean([len(b.txs) for b, _ in wins]))}

    # warm-up: one pass of the loop sizes every per-call buffer of ctx_a; a few mempool calls on both contexts
    s = Setup(ctx_a, wins, prm, fund)
    s.loop()
    mempool_calls(tv_a, s.base, batches, vdaa, 5)
    mempool_calls(tv_b, s.base.on(ctx_b), batches, vdaa, 5)
    ref, diffs = s.statuses, s.diffs
    s.close()

    s = Setup(ctx_a, wins, prm, fund)
    out["alone"] = summary(mempool_calls(tv_b, s.base.on(ctx_b), batches, vdaa, a.calls))
    s.loop(1, diffs)
    out["replay_alone_tx_per_s"] = round(s.tx_per_s)
    s.close()

    def loaded(tv, us_for):
        s = Setup(ctx_a, wins, prm, fund)
        w = threading.Thread(target=s.loop, args=(a.max_passes, diffs))
        w.start()
        ts = mempool_calls(tv, us_for(s), batches, vdaa, a.calls, stop=s)
        w.join()
        assert all((x == y).all() for x, y in zip(s.statuses, ref)), "replay verdicts differ under mempool load"
        r = summary(ts)
        r["replay_tx_per_s"], r["passes"] = round(s.tx_per_s), s.passes
        s.close()
        return r

    out["same_context"] = loaded(tv_a, lambda s: s.base)
    out["shared"] = loaded(tv_b, lambda s: s.base.on(ctx_b))
    hp = torch.cuda.Stream(priority=-1)  # the highest priority torch gives a stream
    ctx_b.use_stream(hp.cuda_stream)
    out["shared_hp"] = loaded(tv_b, lambda s: s.base.on(ctx_b))
    ctx_b.reset_stream()
    ctx_a.close()
    ctx_b.close()
    print("card: %s" % info)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
