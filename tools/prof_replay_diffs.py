"""Device time of kgv_replay_diffs next to kgv_replay_window at the bench's config-3 shape (1024-block windows of the generated
simpa-shaped chain, <= 150 transactions per block, one group per block), the bytes the diff pass moves computed from the shapes, and
kgv_replay_window alone on two builds of the library alternated in one session (to show that recording what the diffs need costs the
window nothing).  Prints one JSON line; needs a GPU.

    python tools/prof_replay_diffs.py [--blocks 3072] [--window 1024] [--reps 3] [--other path/to/libkgv.so]

--other is the build to alternate with (e.g. the parent commit's library); without it only the current build is timed."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rusty_kaspa_b200 import _lib, simgen  # noqa: E402
from rusty_kaspa_b200.replay import REPLAY_BLOCK_DTYPE  # noqa: E402
from rusty_kaspa_b200.validator import Params  # noqa: E402
from rusty_kaspa_b200.verifier import _KgvTxBatch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


class Lib:
    """one build of libkgv.so with its own context, bound to torch's current stream"""

    def __init__(self, path, stream):
        self.path = path
        self.lib = C.CDLL(path)
        for name, res, args in _lib.SYMBOLS:
            fn = getattr(self.lib, name, None)
            if fn is not None:
                fn.restype, fn.argtypes = res, args
        h = C.c_void_p()
        assert self.lib.kgv_create(0, 0, C.byref(h)) == 0
        self.h = h
        assert self.lib.kgv_set_stream(h, C.c_void_p(stream.cuda_stream)) == 0

    def check(self, rc):
        if rc:
            raise RuntimeError("%s: %s" % (self.path, self.lib.kgv_last_error(self.h).decode()))

    def table(self, slots):
        t = C.c_void_p()
        self.check(self.lib.kgv_utxo_create(self.h, slots, C.byref(t)))
        return t

    def close(self):
        self.lib.kgv_destroy(self.h)


def diff_bytes(nt, ni, no, n_groups, n_rem, n_add, n_script):
    """bytes the diff pass reads and writes, from the shapes (records of the window state as laid out in kgv_replay_impl.cuh)"""
    acc_inst = nt * (1 + 16 + 4) + nt * 4                       # accept, tx info, atomicMin; the memset
    groups = (n_groups + 1) * (48 + 72 + 8) + nt * 0 + 4 * (n_groups + 1)
    spender = ni * (4 + 1 + 8 + 4 + 4 + 4) + no * 4             # itx, accept, source, tx->block, block->group, store; the memset
    classify = ni * (4 + 1 + 8 + 4 + 4 + 4 + 32 + 8) + no * (4 + 1 + 16 + 4 + 72 + 4 + 4 + 4 + 24 + 8)
    scan = 2 * (ni + no) * (4 + 8)
    gather = (ni + no) * 4 + n_rem * (4 + 4 + 4 + 8 + 8 + 56 + 32 + 36 + 32) + n_add * (4 + 4 + 4 + 8 + 8 + 32 + 72 + 24 + 16 + 8 + 36 + 32) + 2 * n_script
    return acc_inst + groups + spender + classify + scan + gather


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=3072)
    ap.add_argument("--window", type=int, default=1024)
    ap.add_argument("--tpb", type=int, default=150)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--diff-reps", type=int, default=10)
    ap.add_argument("--other", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    gen = simgen.FastDag(seed=0x6B61737061, n_keys=1024, n_nonces=4096, frac_two_inputs=0.5, frac_invalid=0.01, coinbase_outputs=16)
    wins, done = [], 0
    while done < a.blocks:
        k = min(a.window, a.blocks - done)
        gen.generate(k, a.tpb)
        b, first, pov = gen.take()
        arr = np.zeros(k, dtype=REPLAY_BLOCK_DTYPE)
        arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1
        ts = [torch.from_numpy(x.view(np.uint8).reshape(-1)).to(dev) for x in (b.txs, b.inputs, b.outputs, b.arena)]
        cb = _KgvTxBatch(ts[0].data_ptr(), len(b.txs), ts[1].data_ptr(), len(b.inputs), ts[2].data_ptr(), len(b.outputs), None, ts[3].data_ptr(), len(b.arena))
        wins.append((b, arr, ts, cb, torch.empty(len(b.txs) * 16, dtype=torch.uint8, device=dev)))
        done += k
    prm = Params(coinbase_maturity=gen.maturity, storage_mass_parameter=gen.C)
    libs = [Lib(_lib.LIB_PATH, stream)] + ([Lib(os.path.abspath(a.other), stream)] if a.other else [])
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def run_chain(L, diffs=False):
        """the whole chain on a fresh 2^24-slot table; returns the device ms of every window (and of kgv_replay_diffs after it)"""
        t = L.table(1 << 24)
        w_ms, d_ms, shapes = [], [], []
        for b, arr, ts, cb, dres in wins:
            e0, e1 = ev(), ev()
            e0.record(stream)
            L.check(L.lib.kgv_replay_window(L.h, t, C.byref(cb), arr.ctypes.data, len(arr), C.byref(prm), dres.data_ptr(), None, None))
            e1.record(stream)
            stream.synchronize()
            w_ms.append(e0.elapsed_time(e1))
            if diffs:
                gf = np.arange(len(arr) + 1, dtype=np.uint32)
                rg = torch.empty(len(arr) * 32, dtype=torch.uint8, device=dev)
                nr, na, nb = C.c_size_t(), C.c_size_t(), C.c_size_t()
                L.check(L.lib.kgv_replay_diffs(L.h, gf.ctypes.data, len(arr), rg.data_ptr(), None, None, None, None, None, 0, 0, 0, C.byref(nr), C.byref(na), C.byref(nb)))
                out = [torch.empty(max(x, 1), dtype=torch.uint8, device=dev) for x in (36 * nr.value, 32 * nr.value, 36 * na.value, 32 * na.value, nb.value)]
                times = []
                for _ in range(a.diff_reps):  # steady state: the fill form, device outputs, every call synchronises once (the size check)
                    e2, e3 = ev(), ev()
                    e2.record(stream)
                    L.check(L.lib.kgv_replay_diffs(L.h, gf.ctypes.data, len(arr), rg.data_ptr(), *[o.data_ptr() for o in out], nr.value, na.value, nb.value,
                                                   C.byref(nr), C.byref(na), C.byref(nb)))
                    e3.record(stream)
                    stream.synchronize()
                    times.append(e2.elapsed_time(e3))
                d_ms.append(float(np.median(times[1:])))
                shapes.append((len(b.txs), len(b.inputs), len(b.outputs), len(arr), nr.value, na.value, nb.value))
        L.lib.kgv_utxo_destroy(L.h, t)
        return w_ms, d_ms, shapes

    for L in libs:  # warm-up: sizes every per-call buffer of both contexts
        run_chain(L)
    alt = {L.path: [] for L in libs}
    for _ in range(a.reps):
        for L in libs:
            w_ms, _, _ = run_chain(L)
            alt[L.path].append(sum(w_ms))
    w_ms, d_ms, shapes = run_chain(libs[0], diffs=True)
    per = []
    for (nt, ni, no, ng, nr, na, nb), wm, dm in zip(shapes, w_ms, d_ms):
        by = diff_bytes(nt, ni, no, ng, nr, na, nb)
        per.append({"txs": nt, "inputs": ni, "outputs": no, "blocks": ng, "n_remove": nr, "n_add": na, "script_bytes": nb, "replay_window_ms": round(wm, 3),
                    "replay_diffs_ms": round(dm, 3), "diff_bytes_model": by, "diff_GBps_model": round(by / dm / 1e6, 1)})
    print(json.dumps({"card": card(), "shape": f"config 3: {a.blocks} blocks, <= {a.tpb} txs/block, {a.window}-block windows, one group per block",
                      "windows": per,
                      "replay_window_chain_ms_alternated": {os.path.relpath(k, ROOT): [round(x, 2) for x in v] for k, v in alt.items()}}))
    for L in libs:
        L.close()


if __name__ == "__main__":
    main()
