"""The device script engine on replay windows with a share of declined spends (DESIGN.md §4 "Script engine", §5).

A config-3-shaped window (N blocks x 150 transactions, 50 % 1-in/2-out and 50 % 2-in/2-out, P2PK Schnorr spends of a funded UTXO set) in
which each transaction is, with probability f, a spend of P2SH data envelopes instead (redeem = <pk> CHECKSIG FALSE IF "kasplex" 00 <json>
ENDIF: every input declined by the fast path, one signature check each).  For f in {0, 1 %, 10 %, 50 %}:
  * kgv_replay_window over the window (VERIFY_ONLY blocks, so every repeat sees the same table): wall time, tx/s, n_host_vm, rounds;
  * kgv_check_scripts against kgv_check_scripts_host on the same populated declined set, alternated in one process: median, min, max.
    python tools/prof_script_engine.py [n_blocks=1024] [repeats=5]
"""
import ctypes
import hashlib
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import rusty_kaspa_b200 as rk  # noqa: E402
from rusty_kaspa_b200 import Params  # noqa: E402
from rusty_kaspa_b200.replay import REPLAY_VERIFY_ONLY, DagReplayer, replay_blocks_array  # noqa: E402
from rusty_kaspa_b200.simgen import (DEFAULT_STORAGE_MASS_PARAMETER, SUBNET_COINBASE, SUBNET_NATIVE, SimDag, entries_to_arrays,  # noqa: E402
                                     sighash_all, storage_mass)
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402
from rusty_kaspa_b200.validator import RESULT_DTYPE  # noqa: E402
from rusty_kaspa_b200.verifier import _c_batch  # noqa: E402

TPB = 150
C = DEFAULT_STORAGE_MASS_PARAMETER


def envelope(pk, t):
    body = b'{"p":"krc-20","op":"mint","tick":"T%06d"}' % (t % 1000000)
    redeem = b"\x20" + pk + b"\xac\x00\x63\x07kasplex\x00\x4c" + bytes([len(body)]) + body + b"\x68"
    return redeem, b"\xaa\x20" + hashlib.blake2b(redeem, digest_size=32).digest() + b"\x87"


def window(n_txs, f, seed=7):
    """funded, mutually independent transactions; a share f spends envelopes.  Returns (keys36, entries, txs, declined mask)."""
    dag = SimDag(seed=seed, n_keys=1024, n_nonces=4096, storage_mass_parameter=C)
    rng = dag.rng
    keys, fund, txs, declined = [], [], [], []
    for t in range(n_txs):
        env = rng.random() < f
        n_in = 2 if rng.random() < 0.5 else 1
        ins, ents, meta = [], [], []
        for _ in range(n_in):
            k = int(rng.integers(0, dag.keys.count))
            pk = dag.keys.xs[k]
            redeem, spk = envelope(pk, len(keys)) if env else (None, b"\x20" + pk + b"\xac")
            txid = hashlib.blake2b(len(keys).to_bytes(8, "little") + bytes([seed & 0xFF]), digest_size=32).digest()
            keys.append(txid + bytes(4))
            fund.append({"amount": int(rng.integers(10**8, 10**11)), "spk_version": 0, "script": spk, "block_daa_score": 1, "is_coinbase": False})
            ins.append({"txid": txid, "index": 0, "sigscript": b"", "sequence": 0, "sig_op_count": 1})
            ents.append(fund[-1]); meta.append((k, redeem))
        total = sum(e["amount"] for e in ents)
        outs = [{"value": v, "spk_version": 0, "script": b"\x20" + dag.keys.xs[int(rng.integers(0, dag.keys.count))] + b"\xac"}
                for v in ((total - 1) // 2, total - 1 - (total - 1) // 2)]
        tx = {"version": 0, "inputs": ins, "outputs": outs, "lock_time": 0, "subnetwork_id": SUBNET_NATIVE, "gas": 0, "payload": b"", "mass": 0}
        tx["mass"] = storage_mass([(e["amount"], len(e["script"])) for e in ents], [(o["value"], 34) for o in outs], C)
        for i, (k, redeem) in enumerate(meta):
            sig = b"\x41" + dag._sign(k, sighash_all(tx, ents, i, False), False) + b"\x01"
            ins[i]["sigscript"] = sig + (bytes([0x4C, len(redeem)]) + redeem if redeem else b"")
        txs.append(tx); declined.append(env)
    return np.frombuffer(b"".join(keys), dtype=np.uint8).reshape(-1, 36).copy(), fund, txs, np.array(declined)


def stats(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


def main():
    n_blocks = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    ctx = rk.GpuContext(0)
    lib = ctx._lib
    rounds = ctypes.c_uint32()
    props = __import__("torch").cuda.get_device_properties(0)
    print(f"# {props.name}; {n_blocks} blocks x {TPB} txs; {reps} repeats", flush=True)
    for f in (0.0, 0.01, 0.10, 0.50):
        t0 = time.perf_counter()
        keys, fund, txs, dec = window(n_blocks * TPB, f)
        gen_s = time.perf_counter() - t0
        r = DagReplayer(ctx, Params(coinbase_maturity=0, storage_mass_parameter=C), 1 << 20)
        arr_e, arena = entries_to_arrays(fund)
        r.us.apply_diff(add_keys36=keys, add_entries=arr_e, add_bytes=arena)
        all_txs, ranges = [], []
        for bi in range(n_blocks):
            cb = {"version": 0, "inputs": [], "outputs": [{"value": 5, "spk_version": 0, "script": b"\x51"}], "lock_time": 0, "subnetwork_id": SUBNET_COINBASE,
                  "gas": 0, "payload": b"blk%d" % bi, "mass": 0}
            blk = [cb] + txs[bi * TPB:(bi + 1) * TPB]
            ranges.append((len(all_txs), len(blk), 1000 + bi, REPLAY_VERIFY_ONLY))
            all_txs.extend(blk)
        b, barr = build_batch(all_txs), replay_blocks_array(ranges)
        times = []
        for k in range(reps + 1):
            t0 = time.perf_counter()
            res = r.replay_window(b, barr)
            dt = time.perf_counter() - t0
            if k:
                times.append(dt * 1e3)
        ctx._check(lib.kgv_debug_script_rounds(ctx._h, ctypes.byref(rounds)))
        rr = rounds.value
        nv = r.last_stats["n_host_vm"]
        ok = int((res["status"] == 0).sum())
        assert nv == int(dec.sum()) and ok == len(txs), (nv, int(dec.sum()), ok, len(txs))
        med, lo, hi = stats(times)
        line = (f"f={f:.2f}: {len(all_txs)} txs, {nv} declined; kgv_replay_window {med:.2f} ms (min {lo:.2f}, max {hi:.2f}), "
                f"{len(all_txs) / med * 1e3 / 1e6:.2f} M tx/s, engine rounds {rr}")
        if nv:
            idx_tx = [i for i in range(len(txs)) if dec[i]]
            first = np.concatenate([[0], np.cumsum([len(t["inputs"]) for t in txs])])  # window() appends the funding entries in tx order
            pb = build_batch([txs[i] for i in idx_tx], [fund[first[i]:first[i + 1]] for i in idx_tx])
            idx = np.arange(len(idx_tx), dtype=np.uint32)
            cbb = _c_batch(pb, with_entries=True)
            td, th = [], []
            for k in range(reps + 1):
                for fn, acc in ((lib.kgv_check_scripts, td), (lib.kgv_check_scripts_host, th)):
                    out = np.zeros(len(idx), dtype=RESULT_DTYPE)
                    t0 = time.perf_counter()
                    ctx._check(fn(ctx._h, ctypes.byref(cbb), idx.ctypes.data, len(idx), out.ctypes.data))
                    dt = time.perf_counter() - t0
                    assert (out["status"] == 0).all()
                    if k:
                        acc.append(dt * 1e3)
            ctx._check(lib.kgv_debug_script_rounds(ctx._h, ctypes.byref(rounds)))
            (dm, dl, dh), (hm, hl, hh) = stats(td), stats(th)
            line += (f"; declined set ({len(idx_tx)} txs, {len(pb.inputs)} inputs): kgv_check_scripts {dm:.2f} ms (min {dl:.2f}, max {dh:.2f}), "
                     f"{rounds.value} rounds; kgv_check_scripts_host {hm:.2f} ms (min {hl:.2f}, max {hh:.2f})")
        print(line + f"; generation {gen_s:.0f} s", flush=True)
        r.close()
    ctx.close()


if __name__ == "__main__":
    main()
