"""Cost of kgv_validate_block_bodies.

1. Device-resident time (CUDA events around each call, the calls alternated, median of --reps after --warmup) of kgv_validate_block_bodies
   against the sum of the three calls it replaces on the same data (kgv_block_hash_merkle_roots + kgv_validate_txs_in_isolation +
   kgv_block_set_checks), for a window of 10 000 blocks x 147 transactions (1.47 M transactions, the replay benchmark's window shape) and
   for one block.
2. One body of 50 000 inputs: kgv_block_set_checks, once after a warm-up call, for random outpoints and for outpoints crafted so that the
   UTXO table's public key_hash (kgv_utxo.cuh) is one value for all of them.  --sets-only runs just this part and also works through an
   older build of the library named by KGV_LIB (e.g. one with the pairwise kernel), for comparison.
3. --profile: per-kernel device times of one window call from torch.profiler, in a run of its own, written to --out.
Prints the card's name, power limit and maximum SM clock, read in the same run, and one JSON line.

    python tools/prof_block_bodies.py [--reps 20] [--warmup 3] [--blocks 10000] [--sets-only] [--profile --out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rusty_kaspa_b200 import GpuContext, TxRules  # noqa: E402
from rusty_kaspa_b200.txbatch import INPUT_DTYPE, OUTPUT_DTYPE, TX_DTYPE  # noqa: E402
from rusty_kaspa_b200.validator import BLOCK_HEADER_CTX_DTYPE, BodyRules  # noqa: E402
from rusty_kaspa_b200.verifier import _KgvTxBatch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else "unknown"


def window(n_blocks, txs_per_block, n_in=2, n_out=2, seed=1):
    """valid bodies without per-transaction Python: a coinbase (payload: blue score 7, subsidy 50, no script) and native transactions of
    n_in distinct random outpoints and n_out outputs"""
    rng = np.random.default_rng(seed)
    nt = n_blocks * txs_per_block
    cb = np.arange(nt) % txs_per_block == 0
    T = np.zeros(nt, TX_DTYPE)
    T["n_inputs"] = np.where(cb, 0, n_in)
    T["n_outputs"] = np.where(cb, 1, n_out)
    T["first_input"] = np.cumsum(T["n_inputs"]) - T["n_inputs"]
    T["first_output"] = np.cumsum(T["n_outputs"]) - T["n_outputs"]
    T["subnetwork_id"][cb, 0] = 1
    T["payload_len"] = np.where(cb, 19, 0)
    I = np.zeros(int(T["n_inputs"].sum()), INPUT_DTYPE)
    O = np.zeros(int(T["n_outputs"].sum()), OUTPUT_DTYPE)
    I["prev_txid"] = rng.integers(0, 256, (len(I), 32), dtype=np.uint8)
    I["sigscript_off"], I["sigscript_len"], I["sig_op_count"], I["sequence"] = 64, 66, 1, 2**64 - 1
    O["value"] = rng.integers(1, 10**9, len(O), dtype=np.uint64)
    O["script_off"], O["script_len"] = 64, 34
    arena = np.zeros(256, np.uint8)
    arena[0], arena[8] = 7, 50
    first = (np.arange(n_blocks + 1) * txs_per_block).astype(np.uint32)
    return T, I, O, arena, first


def craft_one_public_hash(I, target=0x0123456789ABCDEF):
    """rewrites the first 8 bytes of every prev_txid so that kgv_utxo.cuh's key_hash is the same for all inputs (they stay distinct)"""
    w = np.ascontiguousarray(I["prev_txid"]).view("<u8").reshape(-1, 4)
    with np.errstate(over="ignore"):
        w[:, 0] = (np.uint64(target) ^ w[:, 1] * np.uint64(0x9E3779B97F4A7C15) ^ w[:, 2] * np.uint64(0xC2B2AE3D27D4EB4F) ^ w[:, 3] * np.uint64(0x165667B19E3779F9)
                   ^ I["prev_index"].astype(np.uint64) * np.uint64(0xD6E8FEB86659FD93))
    I["prev_txid"] = w.view(np.uint8).reshape(-1, 32)
    return I


class Calls:
    def __init__(self, ctx, T, I, O, arena, first):
        import torch
        self.ctx, self.first, self.n, self.nt = ctx, first, len(first) - 1, len(T)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
        self.keep = [dev(a) for a in (T, I, O, arena)]
        t = self.keep
        self.cb = _KgvTxBatch(t[0].data_ptr(), len(T), t[1].data_ptr(), len(I), t[2].data_ptr(), len(O), None, t[3].data_ptr(), len(arena))
        z = lambda n: torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda")
        self.res, self.masses, self.roots, self.txres, self.txm, self.sets = z(self.n * 32), z(self.n * 24), z(self.n * 32), z(self.nt * 16), z(self.nt * 16), z(self.n * 8)
        self.rules, self.body = TxRules(), BodyRules(max_block_mass=2**64 - 1)
        h = np.zeros(self.n, BLOCK_HEADER_CTX_DTYPE)
        h["blue_score"], h["expected_subsidy"], h["daa_score"] = 7, 50, 1000
        self.merkle()
        torch.cuda.synchronize()
        h["hash_merkle_root"] = self.roots.cpu().numpy().reshape(-1, 32)
        self.h = dev(h)

    def merkle(self):
        self.ctx._check(self.ctx._lib.kgv_block_hash_merkle_roots(self.ctx._h, ctypes.byref(self.cb), self.first.ctypes.data, self.n, self.roots.data_ptr()))

    def three_calls(self):
        lib, c = self.ctx._lib, self.ctx
        self.merkle()
        c._check(lib.kgv_validate_txs_in_isolation(c._h, ctypes.byref(self.cb), ctypes.byref(self.rules), 1000, 0, 0, self.txres.data_ptr(), self.txm.data_ptr()))
        self.set_checks()

    def set_checks(self):
        self.ctx._check(self.ctx._lib.kgv_block_set_checks(self.ctx._h, ctypes.byref(self.cb), self.first.ctypes.data, self.n, self.sets.data_ptr()))

    def bodies(self):
        c = self.ctx
        c._check(c._lib.kgv_validate_block_bodies(c._h, ctypes.byref(self.cb), self.first.ctypes.data, self.n, self.h.data_ptr(), ctypes.byref(self.rules),
                                                  ctypes.byref(self.body), 0, self.res.data_ptr(), self.masses.data_ptr(), self.roots.data_ptr()))


def event_ms(fns, reps, warmup):
    """device time of each call, the calls alternated: the median per call"""
    import torch
    for _ in range(warmup):
        for f in fns:
            f()
    t = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            t[k].append(e0.elapsed_time(e1))
    return [float(np.median(x)) for x in t]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=10000)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--sets-only", action="store_true")
    ap.add_argument("--out", default=".")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured without one")
    gpu = card()
    if a.sets_only:  # an older build lacks the newer entry points: bind the ones it has
        from rusty_kaspa_b200 import _lib
        have = ctypes.CDLL(_lib.LIB_PATH)
        _lib.SYMBOLS = [s for s in _lib.SYMBOLS if hasattr(have, s[0])]
    ctx = GpuContext(0)
    ctx.use_torch_stream()
    out = {"gpu": gpu, "unit": "ms of device time per call (median)"}
    if a.profile:
        c = Calls(ctx, *window(a.blocks, 147))
        c.bodies()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            c.bodies()
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=60)
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prof_block_bodies_kernels.txt"), "w") as f:
            f.write("card: %s\n%s\n" % (gpu, table))
        print(table)
    else:
        for name, nb in (("window", a.blocks), ("one block", 1)) if not a.sets_only else ():
            c = Calls(ctx, *window(nb, 147))
            c.bodies()
            torch.cuda.synchronize()
            st = c.res.cpu().numpy().view(np.uint32).reshape(-1, 8)[:, 0]
            assert (st == 0).all(), np.unique(st)
            t_new, t_old = event_ms([c.bodies, c.three_calls], a.reps, a.warmup)
            bytes_in = sum(int(k.numel()) for k in c.keep)
            out[name] = {"blocks": nb, "transactions": c.nt, "kgv_validate_block_bodies": round(t_new, 4), "three_calls": round(t_old, 4),
                         "batch_bytes": bytes_in, "batch_GBps_over_call_time": round(bytes_in / t_new / 1e6, 1)}
            print(f"{name}: {nb} blocks, {c.nt} txs  kgv_validate_block_bodies {t_new:.3f} ms   three calls {t_old:.3f} ms", flush=True)
        out["50000-input body"] = {"library": os.environ.get("KGV_LIB", "in-tree")}
        for name in ("random outpoints", "one public key_hash"):
            T, I, O, arena, first = window(1, 51, n_in=1000, n_out=1)
            c = Calls(ctx, T, craft_one_public_hash(I) if name != "random outpoints" else I, O, arena, first)
            c.set_checks()
            t_sets, = event_ms([c.set_checks], 1, 0)
            assert c.sets.cpu().numpy().view(np.uint32)[0] == 0
            out["50000-input body"][name] = round(t_sets, 4)
            print(f"one body of 50 000 inputs, {name}: kgv_block_set_checks {t_sets:.3f} ms", flush=True)
    print("card:", gpu)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
