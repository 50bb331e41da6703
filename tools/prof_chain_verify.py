"""Cost of kgv_replay_verify_chain against the host composition it replaces, on two windows: the 5 000-block simpa fixture's virtual chain
(1 664 chain blocks in one window) and a generated 1 024-block window (simgen.FastDag, 150-transaction blocks, groups of 2 to 41 blocks).

  device ms    the call with device pointers (it only enqueues) on torch's stream, between two CUDA events on that stream
  call wall    the call with host arrays (ends in one synchronise), host clock
  composition  host clock of what a host does without the call: kgv_replay_muhash + kgv_muhash_prefix_combine + kgv_muhash_finalize_batch
               (check 1), the read-back of the window's tx ids (kgv_tx_ids of the window batch: the ids do not leave the window otherwise) and
               the accepted ids gathered from the accept mask kgv_replay_window returned, kgv_merkle_roots and merkle_hash (check 2), and the
               coinbase check (4) restated on the host (tests/oracle_chain.py: expected_coinbase_transaction and its hash per chain block)
Medians of --reps calls; the card's name and power limit are printed with the numbers.

    python tools/prof_chain_verify.py [--reps 10]
"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def fixture_window(ctx):
    from test_gpu_chain_verify import FIXTURES, Window, _plan, _replayer
    fixture = FIXTURES[1]
    w = Window(fixture, _plan(fixture)[5][1:])
    r = _replayer(ctx, fixture)
    w.replay(r)
    txs = [b["txs"] for b in w.blocks]
    return r, w.batch, np.array(w.first + [w.batch.n_txs], np.int64), w.res, w.acc, np.array(w.group_first), w.headers, w.merged_flags(), txs


def generated_window(ctx):
    from rusty_kaspa_b200 import Params, simgen
    from rusty_kaspa_b200.replay import CHAIN_HEADER_DTYPE, REPLAY_ACCEPT_COINBASE, REPLAY_BLOCK_DTYPE, REPLAY_VERIFY_ONLY, DagReplayer
    g = simgen.FastDag(seed=41, n_keys=256, n_nonces=1024, coinbase_maturity=3, frac_invalid=0.02, coinbase_outputs=16)
    # groups of 2 to 41 blocks; each chain block's own body (the VERIFY_ONLY tail) carries 2 transactions, so that few generated outputs
    # go missing for the blocks after it
    gf, sizes = [0], [2, 5, 41, 12, 34, 3, 40]
    while gf[-1] < 1024:
        s = min(sizes[len(gf) % len(sizes)], max(1024 - gf[-1], 2))
        g.generate(s - 1, 150)
        g.generate(1, 2)
        gf.append(gf[-1] + s)
    b, first, pov = g.take()
    nb = len(pov)
    # every merged block's coinbase is accepted (the generator spends them later); only the selected parent's id counts (ctx.accepted_tx_ids)
    flags = np.full(nb, REPLAY_ACCEPT_COINBASE, np.uint32)
    flags[np.array(gf[1:]) - 1] = REPLAY_VERIFY_ONLY
    arr = np.zeros(nb, dtype=REPLAY_BLOCK_DTYPE)
    arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, flags
    r = DagReplayer(ctx, Params(coinbase_maturity=3, storage_mass_parameter=g.C), 1 << 20)
    res, acc = r.replay_window(b, arr, want_accept=True)
    g.close()
    return r, b, np.asarray(first, np.int64), res, acc, np.array(gf), np.zeros(len(gf) - 1, dtype=CHAIN_HEADER_DTYPE), np.zeros(nb, np.uint8), None


def coinbase_payload(batch, t):
    tx = batch.txs[t]
    return batch.arena[int(tx["payload_off"]):int(tx["payload_off"]) + int(tx["payload_len"])].tobytes()


def host_coinbase_check(batch, first, res, acc, gf, headers, mflags, txs):
    """check 4 restated on the host, per chain block (the rewards from the window's fees and accept mask, payloads from the batch)"""
    import oracle_chain as oc
    import pyref
    n_ok = 0
    for g in range(len(gf) - 1):
        b0, bt = int(gf[g]), int(gf[g + 1]) - 1
        try:
            rewards = []
            for k in range(b0, bt):
                lo, hi = int(first[k]), int(first[k + 1])
                _, ver, script, _ = oc.miner_data(coinbase_payload(batch, lo), 204, 150)
                sub = int.from_bytes(coinbase_payload(batch, lo)[8:16], "little")
                rewards.append((sub, int(res["fee"][lo + 1:hi][acc[lo + 1:hi] == 1].sum()), ver, script, int(mflags[k])))
            h = headers[g]
            cb = oc.expected_coinbase_transaction(rewards, int(h["blue_score"]), int(h["expected_subsidy"]), coinbase_payload(batch, int(first[bt])), 204, 150)
            n_ok += pyref.tx_hash(cb) == pyref.tx_hash(txs[bt][0])
        except oc.ChainPanic:
            pass
    return n_ok


def measure(ctx, name, r, batch, first, res, acc, gf, headers, mflags, txs, reps):
    import torch
    import pyref
    from rusty_kaspa_b200.muhash import MuHash, finalize_batch, prefix_combine
    from rusty_kaspa_b200.validator import BodyRules, TxRules
    init = MuHash(ctx)
    lib, h = ctx._lib, ctx._h
    n_groups, nb = len(gf) - 1, len(mflags)
    rules, body = TxRules(), BodyRules()
    gfa = np.ascontiguousarray(gf, dtype=np.uint32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    dh, dmf, dinit = dev(headers), dev(mflags), dev(np.frombuffer(init.numerator + init.denominator, dtype=np.uint8))
    dres, dfee, dms = (torch.zeros(n, dtype=torch.uint8, device="cuda") for n in (n_groups * 112, nb * 8, n_groups * 768))
    torch.cuda.synchronize()
    t_dev, t_wall, t_mu, t_merkle, t_cb = [], [], [], [], []
    for _ in range(reps + 1):
        # device time: the call with device pointers only enqueues; on torch's stream, two events bracket its work on the device
        ctx.use_torch_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ctx._check(lib.kgv_replay_verify_chain(h, gfa.ctypes.data, n_groups, dh.data_ptr(), dmf.data_ptr(), dinit.data_ptr(), ctypes.byref(rules), ctypes.byref(body),
                                               dres.data_ptr(), dfee.data_ptr(), dms.data_ptr()))
        e1.record()
        torch.cuda.synchronize()
        ctx.reset_stream()
        t_dev.append(e0.elapsed_time(e1))
        t = time.perf_counter()
        r.verify_chain(gf, headers, mflags, init)
        t_wall.append(1e3 * (time.perf_counter() - t))
        t = time.perf_counter()
        finalize_batch(ctx, prefix_combine(ctx, r.replay_muhash(gf), init))
        t_mu.append(1e3 * (time.perf_counter() - t))
    # the rest of the composition stages another batch (the tx ids), which ends the window: timed after the window's own calls
    for _ in range(reps + 1):
        t = time.perf_counter()
        ids = ctx.tx_ids(batch)
        sel, off = [], [0]
        for g in range(n_groups):
            b0, bt = int(gf[g]), int(gf[g + 1]) - 1
            keep = [int(first[b0])] + [t2 for k in range(b0, bt) for t2 in range(int(first[k]) + 1, int(first[k + 1])) if acc[t2]]
            sel += keep
            off.append(len(sel))
        roots = ctx.merkle_roots(ids[np.array(sel)], off)
        for g in range(n_groups):
            pyref.blake2b_keyed(b"MerkleBranchHash", headers[g]["selected_parent_accepted_id_merkle_root"].tobytes() + roots[g].tobytes())
        t_merkle.append(1e3 * (time.perf_counter() - t))
        t = time.perf_counter()
        host_coinbase_check(batch, first, res, acc, gf, headers, mflags, txs if txs is not None else [[{"outputs": []}]] * nb)
        t_cb.append(1e3 * (time.perf_counter() - t))
    med = lambda a: float(np.median(a[1:]))
    comp = med(t_mu) + med(t_merkle) + med(t_cb)
    print("%s: %d chain blocks, %d window blocks, %d transactions" % (name, n_groups, nb, batch.n_txs))
    print("  kgv_replay_verify_chain   device %.3f ms   call wall (host arrays) %.3f ms" % (med(t_dev), med(t_wall)))
    print("  composition (host clock)  %.3f ms = MuHash calls %.3f + tx ids / accepted ids / merkle roots %.3f + host coinbase check %.3f"
          % (comp, med(t_mu), med(t_merkle), med(t_cb)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import rusty_kaspa_b200 as rk
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card: %s" % card)
    ctx = rk.GpuContext(0)
    for name, make in (("5 000-block fixture", fixture_window), ("generated 1 024-block window", generated_window)):
        r, *rest = make(ctx)
        measure(ctx, name, r, *rest, args.reps)
        r.close()
    ctx.close()


if __name__ == "__main__":
    main()
