"""kgv_replay_diffs: the UtxoDiff of every group of blocks of a replay window (ctx.mergeset_diff of calculate_utxo_state), checked against
diffs built on the CPU with utxo_diff.UtxoDiff.add_transaction over a block-by-block oracle replay, against the reference's own header
commitments (rollback and roll-forward over the simpa fixtures), and through a reorg on a view layer."""
import copy
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle_tx
from rusty_kaspa_b200 import KgvError, MuHash, Params
from rusty_kaspa_b200.replay import (DagReplayer, REPLAY_ACCEPT_COINBASE, REPLAY_SKIP_SCRIPTS, REPLAY_VERIFY_ONLY, replay_blocks_array)
from rusty_kaspa_b200.simgen import FastDag, SimDag, tx_id
from rusty_kaspa_b200.txbatch import TxBatch, build_batch
from rusty_kaspa_b200.utxo_diff import UtxoDiff

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ CPU side
def _slice(b, t0, t1):
    """transactions [t0, t1) of a batch as a batch of their own (same arena)"""
    T = b.txs[t0:t1].copy()
    if t1 == t0:
        return TxBatch(T, b.inputs[:0].copy(), b.outputs[:0].copy(), None, b.arena)
    i0, i1 = int(T[0]["first_input"]), int(T[-1]["first_input"] + T[-1]["n_inputs"])
    o0, o1 = int(T[0]["first_output"]), int(T[-1]["first_output"] + T[-1]["n_outputs"])
    T["first_input"] -= i0
    T["first_output"] -= o0
    return TxBatch(T, b.inputs[i0:i1].copy(), b.outputs[o0:o1].copy(), None, b.arena)


class CpuReplay:
    """Block-by-block oracle replay that records, per block, the accepted transactions with the entries their inputs spent
    (State.get before the block is applied): enough to build the reference UtxoDiff of any grouping of the blocks."""

    def __init__(self, oracle, op):
        self.oracle, self.op, self.ost = oracle, op, oracle_tx.State(oracle)
        self.blocks = []  # per block: list of (tx dict, entries, txid, pov, is_coinbase); plus per block input / output keys in window order
        self.results, self.accept = [], []

    def close(self):
        self.ost.close()

    def block(self, b, pov, flags):
        ids = oracle_tx.tx_ids(self.oracle, b)
        keys = [b.inputs[i]["prev_txid"].tobytes() + int(b.inputs[i]["prev_index"]).to_bytes(4, "little") for i in range(len(b.inputs))]
        before = [self.ost.get(k) for k in keys]
        res, acc = oracle_tx.state_replay(self.ost, b, np.array([0, len(b.txs)], np.uint32), np.array([pov], np.uint64), self.op,
                                          block_flags=np.array([flags], np.uint32), threads=2)
        rec = []
        for ti in range(len(b.txs)):
            if not acc[ti]:
                continue
            t = b.txs[ti]
            i0, n_in, o0, n_out = int(t["first_input"]), int(t["n_inputs"]), int(t["first_output"]), int(t["n_outputs"])
            txd = {"inputs": [{"txid": keys[i][:32], "index": int.from_bytes(keys[i][32:], "little")} for i in range(i0, i0 + n_in)],
                   "outputs": [{"value": int(o["value"]), "spk_version": int(o["spk_version"]),
                                "script": b.arena[int(o["script_off"]):int(o["script_off"]) + int(o["script_len"])].tobytes()} for o in b.outputs[o0:o0 + n_out]]}
            ents = before[i0:i0 + n_in]
            assert all(e is not None for e in ents)
            rec.append((txd, ents, ids[ti].tobytes(), pov, ti == 0 or bool(t["flags"] & 1)))
        self.blocks.append(rec)
        self.results.append(res)
        self.accept.append(acc)

    def window(self, b, first, pov, flags):
        for k in range(len(pov)):
            self.block(_slice(b, int(first[k]), int(first[k + 1])), int(pov[k]), int(flags[k]))

    def diffs(self, group_first, base=0):
        """expected UtxoDiff per group (blocks numbered from `base`), plus the removal / addition outpoints in window order"""
        out = []
        for g in range(len(group_first) - 1):
            d, rem_order, add_order = UtxoDiff(), [], []
            for bi in range(base + group_first[g], base + group_first[g + 1]):
                for txd, ents, tid, pov, cb in self.blocks[bi]:
                    d.add_transaction(txd, ents, tid, pov, is_coinbase=cb)
                    rem_order += [(i["txid"], i["index"]) for i in txd["inputs"]]
                    add_order += [(tid, k) for k in range(len(txd["outputs"]))]
            out.append((d, [o for o in rem_order if o in d.remove], [o for o in add_order if o in d.add]))
        return out


def _flat(blocks, flags=None):
    """list of (txs, pov) -> (batch, block_first_tx, pov, flags)"""
    txs, first, pov = [], [0], []
    for t, p in blocks:
        txs += t
        first.append(len(txs))
        pov.append(p)
    fl = np.full(len(blocks), REPLAY_ACCEPT_COINBASE, np.uint32) if flags is None else np.asarray(flags, np.uint32)
    return build_batch(txs), np.array(first, np.uint32), np.array(pov, np.uint64), fl


def _blocks_arr(first, pov, flags):
    return replay_blocks_array((int(first[k]), int(first[k + 1] - first[k]), int(pov[k]), int(flags[k])) for k in range(len(pov)))


def _keys(arr):
    return [(k[:32].tobytes(), int.from_bytes(k[32:].tobytes(), "little")) for k in arr]


def _check_against_cpu(got, exp):
    """GPU ReplayDiffs vs [(UtxoDiff, rem_order, add_order)]: equal as dicts, and in window order"""
    assert len(got) == len(exp)
    for g, (d, rem_order, add_order) in enumerate(exp):
        assert got.utxo_diff(g) == d, g
        rk, _, ak, _ = got.group(g)
        assert _keys(rk) == rem_order and _keys(ak) == add_order, g
    # groups are contiguous ranges, in order
    fr, nr, fa, na = got.ranges.T.astype(np.int64) if len(got) else (0, 0, 0, 0)
    assert (fr[1:] == fr[:-1] + nr[:-1]).all() and (fa[1:] == fa[:-1] + na[:-1]).all()
    assert fr[0] == 0 and fa[0] == 0 and fr[-1] + nr[-1] == len(got.rem_keys36) and fa[-1] + na[-1] == len(got.add_keys36)


def _fold(diffs):
    acc = UtxoDiff()
    for d in diffs:
        acc = acc.with_diff(d)
    return acc


def _groupings(n_blocks, rng):
    out = [np.arange(n_blocks + 1), np.array([0, n_blocks])]
    cuts = np.sort(rng.integers(0, n_blocks + 1, size=max(2, n_blocks // 5)))
    out.append(np.concatenate([[0], cuts, cuts[:2], [n_blocks, n_blocks]]).astype(np.int64))  # repeated cuts = empty groups
    out[-1].sort()
    return [g.astype(np.uint32) for g in out]


# ------------------------------------------------------------------------------------------------ 1. generated chains
def test_generated_chains_match_the_cpu_diffs_for_every_grouping(gpu_ctx, oracle):
    g = FastDag(seed=41, n_keys=64, n_nonces=256, coinbase_maturity=2, mix=(0.4, 0.2, 0.2, 0.2), frac_invalid=0.05, coinbase_outputs=8)
    prm = Params(coinbase_maturity=2, storage_mass_parameter=g.C)
    cpu = CpuReplay(oracle, oracle_tx.params(coinbase_maturity=2, storage_mass_parameter=g.C))
    r = DagReplayer(gpu_ctx, prm, 1 << 16)
    rng = np.random.default_rng(8)
    n_in_window_spends = base = 0
    for _ in range(3):
        g.generate(30, 24)
        b, first, pov = g.take()
        flags = np.full(len(pov), REPLAY_ACCEPT_COINBASE, np.uint32)
        res, acc = r.replay_window(b, _blocks_arr(first, pov, flags), want_accept=True)
        cpu.window(b, first, pov, flags)
        assert (acc == np.concatenate(cpu.accept[base:])).all()
        per_block = None
        for gf in _groupings(len(pov), rng):
            got = r.replay_diffs(gf)
            exp = cpu.diffs(gf, base)
            _check_against_cpu(got, exp)
            if len(gf) == len(pov) + 1:
                per_block = [got.utxo_diff(k) for k in range(len(got))]
            if len(gf) == 2:
                whole = got.utxo_diff(0)
                assert _fold(per_block) == whole
                # outputs created in one block and spent in a later one of the window are in neither list of the whole-window diff
                inner = set().union(*(d.add.keys() for d in per_block)) & set().union(*(d.remove.keys() for d in per_block))
                assert not inner & (whole.add.keys() | whole.remove.keys())
                n_in_window_spends += len(inner)
        base += len(pov)
    assert n_in_window_spends > 50, n_in_window_spends
    r.close(); cpu.close(); g.close()


# ------------------------------------------------------------------------------------------------ 2. block flags
def test_block_flags(gpu_ctx, oracle):
    dag = SimDag(seed=19, n_keys=64, n_nonces=128, mix=(0.5, 0.2, 0.2, 0.1), frac_invalid=0.0, coinbase_maturity=2, coinbase_outputs=6)
    blocks = [dag.make_block(10) for _ in range(24)]
    # one transaction with a broken signature in a SkipScriptChecks block: accepted there, so it is in the diff
    bad_b = 9
    bad = blocks[bad_b][0][3]
    ss = bytearray(bad["inputs"][0]["sigscript"])
    ss[10] ^= 0x40
    bad["inputs"][0]["sigscript"] = bytes(ss)
    # (everything before the SkipScriptChecks block applies normally, so the broken transaction's inputs exist)
    flags = np.array([1] * 9 + [3, 1, 0, 1, 4, 1, 5, 1, 2, 1, 4, 0, 3, 1, 1], np.uint32)
    b, first, pov, fl = _flat(blocks, flags)
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    cpu = CpuReplay(oracle, oracle_tx.params(coinbase_maturity=2, storage_mass_parameter=dag.C))
    cpu.window(b, first, pov, fl)
    r = DagReplayer(gpu_ctx, prm, 1 << 14)
    res, acc = r.replay_window(b, _blocks_arr(first, pov, fl), want_accept=True)
    assert (acc == np.concatenate(cpu.accept)).all()
    gf = np.arange(len(pov) + 1, dtype=np.uint32)
    got = r.replay_diffs(gf)
    _check_against_cpu(got, cpu.diffs(gf))
    ids = oracle_tx.tx_ids(oracle, b)
    for k in range(len(pov)):
        d = got.utxo_diff(k)
        cb_outs = {(ids[first[k]].tobytes(), j) for j in range(len(blocks[k][0][0]["outputs"]))}
        if fl[k] & REPLAY_VERIFY_ONLY:
            assert not d.add and not d.remove, k
        elif not fl[k] & REPLAY_ACCEPT_COINBASE:
            assert not (cb_outs & d.add.keys()), k
        else:
            assert cb_outs <= d.add.keys(), k
    assert fl[bad_b] & REPLAY_SKIP_SCRIPTS
    d = got.utxo_diff(bad_b)
    assert (tx_id(bad), 0) in d.add and (bad["inputs"][0]["txid"], bad["inputs"][0]["index"]) in d.remove
    r.close(); cpu.close()


# ------------------------------------------------------------------------------------------------ 3. what only a DAG window holds
def _dag_window():
    """sibling duplicates, a double spend by a different transaction, a copy placed before its original, broken creators
    (built as in test_gpu_replay.py's sibling-duplicate test)"""
    dag = SimDag(seed=77, n_keys=64, n_nonces=128, mix=(0.6, 0.2, 0.1, 0.1), frac_invalid=0.0, coinbase_maturity=2, coinbase_outputs=6)
    rng = np.random.default_rng(3)
    blocks = []
    for bi in range(42):
        before = {(u["txid"], u["index"]): u for u in dag.utxos}
        txs, pov = dag.make_block(14)
        blocks.append((list(txs), pov))
        if bi in (10, 20, 30):
            left = {(u["txid"], u["index"]) for u in dag.utxos}
            cand = [u for k, u in before.items() if k not in left and not u["coinbase"] and u["amount"] >= 4]
            saved, dag.utxos = dag.utxos, [cand[0]]
            txs2, pov2 = dag.make_block(1)
            blocks.append((list(txs2), pov2))
            dag.utxos = saved + dag.utxos
    dups = ((5, 6, 2), (5, 9, 2), (12, 13, 4), (17, 25, 1), (31, 28, 3), (34, 35, 5), (34, 36, 5))
    instances = []  # per duplicated transaction: its id and both (block, position)
    for src_b, dst_b, k in dups:
        instances.append((tx_id(blocks[src_b][0][k]), [(src_b, k), (dst_b, len(blocks[dst_b][0]))]))
        blocks[dst_b][0].append(copy.deepcopy(blocks[src_b][0][k]))
    ids = {}
    for bi, (txs, _) in enumerate(blocks):
        for ti, t in enumerate(txs):
            ids.setdefault(tx_id(t), (bi, ti))
    broken = 0
    for bi in range(len(blocks) - 1, 0, -1):
        for t in blocks[bi][0][1:]:
            src = ids.get(t["inputs"][0]["txid"])
            if src and src[1] > 0 and broken < 5 and rng.random() < 0.5:
                c = blocks[src[0]][0][src[1]]
                ss = bytearray(c["inputs"][0]["sigscript"])
                if len(ss) > 20 and ss[10] == c["inputs"][0]["sigscript"][10]:
                    ss[10] ^= 0x40
                    c["inputs"][0]["sigscript"] = bytes(ss)
                    broken += 1
    assert broken >= 3
    return dag, blocks, instances


def test_dag_window_with_siblings_double_spends_and_broken_creators(gpu_ctx, oracle):
    dag, blocks, instances = _dag_window()
    b, first, pov, fl = _flat(blocks)
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    cpu = CpuReplay(oracle, oracle_tx.params(coinbase_maturity=2, storage_mass_parameter=dag.C))
    cpu.window(b, first, pov, fl)
    statuses = np.concatenate([x["status"] for x in cpu.results])
    assert (statuses == 1).sum() >= len(instances)
    # a transaction several blocks carry: its outputs land in the group of the instance that was accepted (the copy placed before its original
    # included), and nowhere else
    owner = {}
    for tid, inst in instances:
        acc = [(bi, ti) for bi, ti in inst if cpu.accept[bi][ti]]
        assert len(acc) <= 1
        if acc:
            owner[tid] = acc[0][0]
    assert len(owner) >= 4
    for piece in (len(blocks), 7):
        r = DagReplayer(gpu_ctx, prm, 1 << 14)
        n_owned = 0
        for w in range(0, len(blocks), piece):
            n = min(piece, len(blocks) - w)
            sub = _flat(blocks[w:w + n])
            r.replay_window(sub[0], _blocks_arr(*sub[1:]))
            gf = np.arange(n + 1, dtype=np.uint32)
            got = r.replay_diffs(gf)
            _check_against_cpu(got, cpu.diffs(gf, w))
            for tid, bi in owner.items():
                for k in range(n):
                    assert ((tid, 0) in got.utxo_diff(k).add) == (k == bi - w), (tid.hex(), bi, w + k)
                n_owned += w <= bi < w + n
            # the whole piece as one group equals the fold of its blocks
            whole = r.replay_diffs(np.array([0, n], np.uint32))
            assert whole.utxo_diff(0) == _fold(got.utxo_diff(k) for k in range(n))
        assert n_owned == len(owner)
        r.close()
    cpu.close()


# ------------------------------------------------------------------------------------------------ 4. rollback against the reference's headers
@pytest.mark.parametrize("fixture,check_every", [("simpa_goref_1060.json.gz", 1), ("simpa_goref_pruning_5000.json.gz", 64)])
def test_rollback_and_roll_forward_reproduce_every_header_commitment(gpu_ctx, fixture, check_every):
    from golden_util import simpa_dag_replay_plan
    fx, by, order, sp, ordered_mergeset, chain = simpa_dag_replay_plan(fixture)
    txs, ranges, group_first = [], [], [0]
    for blk in chain[1:]:
        pov = by[blk]["daa_score"]
        for k, mb in enumerate(ordered_mergeset(blk)):
            t = by[mb]["txs"]
            ranges.append((len(txs), len(t), pov, (REPLAY_ACCEPT_COINBASE | REPLAY_SKIP_SCRIPTS) if k == 0 else 0))
            txs.extend(t)
        group_first.append(len(ranges))
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=fx["coinbase_maturity"], storage_mass_parameter=fx["storage_mass_parameter"]), 1 << 16)
    r.replay_window(build_batch(txs), replay_blocks_array(ranges))
    diffs = r.replay_diffs(group_first)
    n = len(diffs)
    assert n == len(chain) - 1 > 30
    want = [by[blk].get("utxo_commitment") for blk in chain]  # want[g + 1]: after chain block g of the window
    commit = lambda: MuHash.of_utxo_set(gpu_ctx, r.us).finalize().hex()
    assert commit() == want[n]
    # walk back from the tip: reversed diffs, tip first
    for g in range(n - 1, -1, -1):
        rs, as_ = diffs.apply(r.us, g, reverse=True)
        assert (rs == 1).all() and (as_ == 1).all(), g
        if g > 0 and (g % check_every == 0 or g == 1):
            assert commit() == want[g], g
    assert r.us.count() == 0
    from rusty_kaspa_b200 import GpuUtxoSet
    e = GpuUtxoSet(gpu_ctx, 1 << 10)
    assert r.us.digest() == e.digest()
    e.close()
    # and forward again to the tip
    for g in range(n):
        rs, as_ = diffs.apply(r.us, g)
        assert (rs == 1).all() and (as_ == 1).all(), g
        if g % check_every == 0:
            assert commit() == want[g + 1], g
    assert commit() == want[n]
    r.close()


# ------------------------------------------------------------------------------------------------ 5. reorg on a view
def test_reorg_on_a_view_equals_a_fresh_replay_of_the_new_branch(gpu_ctx, oracle):
    dag = SimDag(seed=5, n_keys=64, n_nonces=128, mix=(0.5, 0.2, 0.2, 0.1), frac_invalid=0.04, coinbase_maturity=2, coinbase_outputs=6)
    prefix = [dag.make_block(12) for _ in range(16)]
    fork = copy.deepcopy(dag)
    fork.rng = np.random.default_rng(1234)
    a0 = dag.make_block(12)
    cb_a = a0[0][0]
    ida = tx_id(cb_a)
    cb_utxos = [dict(u) for u in dag.utxos if u["txid"] == ida]
    branch_a = [a0] + [dag.make_block(12) for _ in range(7)]
    # both branches' first blocks carry the SAME coinbase (same outpoints, same DAA score): the reorg removes and re-adds them
    b0 = fork.make_block(12)
    idb = tx_id(b0[0][0])
    assert b0[1] == a0[1] and idb != ida and len(cb_utxos) == len(cb_a["outputs"])
    fork.utxos = [u for u in fork.utxos if u["txid"] != idb] + cb_utxos
    branch_b = [([cb_a] + b0[0][1:], b0[1])] + [fork.make_block(12) for _ in range(9)]
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)

    def windows(rep, blocks, size):
        res = []
        for w in range(0, len(blocks), size):
            sub = _flat(blocks[w:w + size])
            res.append(rep.replay_window(sub[0], _blocks_arr(*sub[1:])))
        return res

    # P + A into a table, collecting A's diffs (one group per block, two windows)
    r = DagReplayer(gpu_ctx, prm, 1 << 14)
    windows(r, prefix, 8)
    a_diffs = []
    for w in range(0, len(branch_a), 5):
        sub = _flat(branch_a[w:w + 5])
        r.replay_window(sub[0], _blocks_arr(*sub[1:]))
        a_diffs.append(r.replay_diffs(np.arange(len(sub[2]) + 1, dtype=np.uint32)))
    assert r.us.count() > 0
    # the reorg: a view over the table, A's diffs reversed tip first, B replayed windowed on the view, then committed
    view = r.us.compose(1 << 14)
    n_cb_removed = 0
    for d in reversed(a_diffs):
        for g in range(len(d) - 1, -1, -1):
            rs, as_ = d.apply(view, g, reverse=True)
            assert (rs == 1).all() and (as_ == 1).all()
            n_cb_removed += sum(1 for k in _keys(d.group(g)[2]) if k[0] == ida)
    assert n_cb_removed == len(cb_a["outputs"])
    base = r.us
    r.us = view
    got_b = windows(r, branch_b, 4)
    b_diffs_view = r.replay_diffs(np.arange(len(branch_b[8:]) + 1, dtype=np.uint32))
    view.commit()
    r.us = base
    # a fresh replay of P + B
    f = DagReplayer(gpu_ctx, prm, 1 << 14)
    windows(f, prefix, 8)
    exp_b = windows(f, branch_b, 4)
    b_diffs_fresh = f.replay_diffs(np.arange(len(branch_b[8:]) + 1, dtype=np.uint32))
    for x, y in zip(got_b, exp_b):
        assert (x["status"] == y["status"]).all() and (x["script_err"] == y["script_err"]).all() and (x["fee"] == y["fee"]).all()
    assert all(b_diffs_view.utxo_diff(k) == b_diffs_fresh.utxo_diff(k) for k in range(len(b_diffs_fresh)))
    assert r.us.count() == f.us.count() and r.us.digest() == f.us.digest()
    assert MuHash.of_utxo_set(gpu_ctx, r.us).finalize() == MuHash.of_utxo_set(gpu_ctx, f.us).finalize()
    statuses = np.concatenate([x["status"] for x in got_b])
    assert (statuses == 0).sum() > 50
    view.close(); r.close(); f.close()


# ------------------------------------------------------------------------------------------------ 6. contract
def _raw(ctx, gf, ranges=None, arrays=None, caps=(0, 0, 0)):
    lib = ctx._lib
    nr, na, nb = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    rk, re, ak, ae, by = arrays if arrays is not None else (None,) * 5
    gfa = np.ascontiguousarray(gf, np.uint32)
    rc = lib.kgv_replay_diffs(ctx._h, gfa.ctypes.data, len(gfa) - 1, ranges, rk, re, ak, ae, by, caps[0], caps[1], caps[2], ctypes.byref(nr), ctypes.byref(na),
                              ctypes.byref(nb))
    return rc, (nr.value, na.value, nb.value)


def test_contract_sizes_errors_order_independence_and_device_outputs(gpu_ctx, oracle):
    import torch
    dag = SimDag(seed=23, n_keys=32, n_nonces=64, mix=(0.6, 0.2, 0.1, 0.1), frac_invalid=0.05, coinbase_maturity=2, coinbase_outputs=4)
    blocks = [dag.make_block(10) for _ in range(12)]
    b, first, pov, fl = _flat(blocks)
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=2, storage_mass_parameter=dag.C), 1 << 14)
    # no window yet in this state: staging any batch ends the window the call would refer to
    r.replay_window(b, _blocks_arr(first, pov, fl))
    gpu_ctx.tx_ids(b)
    assert _raw(gpu_ctx, [0, len(pov)])[0] == -1
    with pytest.raises(KgvError):
        r.replay_diffs([0, len(pov)])
    r.close()
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=2, storage_mass_parameter=dag.C), 1 << 14)
    r.replay_window(b, _blocks_arr(first, pov, fl))
    gf = np.array([0, 3, 3, 7, len(pov)], np.uint32)
    # groups that do not tile the window
    for bad in ([0, 3, len(pov) - 1], [1, 3, len(pov)], [0, 5, 3, len(pov)], [0, len(pov) + 1]):
        assert _raw(gpu_ctx, bad)[0] == -1, bad
    # MuHash alone, then diffs, then MuHash again (and diffs again): nothing changes
    mu0 = r.replay_muhash(gf)
    d1 = r.replay_diffs(gf)
    mu1 = r.replay_muhash(gf)
    d2 = r.replay_diffs(gf)
    assert (mu0 == mu1).all()
    for x, y in ((d1.ranges, d2.ranges), (d1.rem_keys36, d2.rem_keys36), (d1.rem_entries, d2.rem_entries), (d1.add_keys36, d2.add_keys36),
                 (d1.add_entries, d2.add_entries), (d1.bytes, d2.bytes)):
        assert x.tobytes() == y.tobytes()
    # size query, then arrays one row / one byte too small: KGV_ERR_NOMEM with the sizes set
    rc, (nr, na, nb) = _raw(gpu_ctx, gf)
    assert rc == 0 and (nr, na, nb) == (len(d1.rem_keys36), len(d1.add_keys36), len(d1.bytes)) and nr > 0 and na > 0
    host = [np.zeros(36 * nr), np.zeros(32 * nr), np.zeros(36 * na), np.zeros(32 * na), np.zeros(nb + 8)]
    ptrs = tuple(a.ctypes.data for a in host)
    for caps in ((nr - 1, na, nb), (nr, na - 1, nb), (nr, na, nb - 1)):
        rg = np.zeros((len(gf) - 1, 4), np.uint64)
        rc, sizes = _raw(gpu_ctx, gf, rg.ctypes.data, ptrs, caps)
        assert rc == -3 and sizes == (nr, na, nb) and (rg == d1.ranges).all()
    # the muhash still matches after all of this
    assert (r.replay_muhash(gf) == mu0).all()
    # device outputs equal host outputs
    dev = torch.device("cuda", 0)
    t = [torch.zeros(max(x, 1), dtype=torch.uint8, device=dev) for x in (36 * nr + 1, 32 * nr, 36 * na + 3, 32 * na, nb)]
    rg = torch.zeros((len(gf) - 1) * 32, dtype=torch.uint8, device=dev)
    # (keys at an odd offset: the key arrays need no alignment)
    rc, sizes = _raw(gpu_ctx, gf, rg.data_ptr(), (t[0].data_ptr() + 1, t[1].data_ptr(), t[2].data_ptr() + 3, t[3].data_ptr(), t[4].data_ptr()), (nr, na, nb))
    torch.cuda.synchronize()
    assert rc == 0 and sizes == (nr, na, nb)
    assert rg.cpu().numpy().tobytes() == d1.ranges.tobytes()
    assert t[0].cpu().numpy()[1:].tobytes() == d1.rem_keys36.tobytes() and t[1].cpu().numpy().tobytes() == d1.rem_entries.tobytes()
    assert t[2].cpu().numpy()[3:].tobytes() == d1.add_keys36.tobytes() and t[3].cpu().numpy().tobytes() == d1.add_entries.tobytes()
    assert t[4].cpu().numpy()[:nb].tobytes() == d1.bytes.tobytes()
    r.close()


# ------------------------------------------------------------------------------------------------ 7. C++ mirror
def test_cpp_mirror_prints_the_same_diffs(gpu_ctx, tmp_path):
    src = os.path.join(ROOT, "tests", "cpp", "replay_diffs_test.cpp")
    exe = str(tmp_path / "replay_diffs_test")
    libdir = os.path.join(ROOT, "rusty_kaspa_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, src, "-L" + libdir, "-l:libkgv.so", "-Wl,-rpath," + libdir], check=True)
    dag = SimDag(seed=61, n_keys=32, n_nonces=64, mix=(0.5, 0.2, 0.2, 0.1), frac_invalid=0.05, coinbase_maturity=2, coinbase_outputs=4)
    b, first, pov, fl = _flat([dag.make_block(8) for _ in range(14)])
    d = str(tmp_path)
    for name, arr in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("arena", b.arena), ("blocks", _blocks_arr(first, pov, fl))):
        arr.tofile(os.path.join(d, name + ".bin"))
    gf = np.array([0, 1, 4, 4, 9, 14], np.uint32)
    gf.tofile(os.path.join(d, "groups.bin"))
    out = subprocess.run([exe, d, "2", str(dag.C)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=2, storage_mass_parameter=dag.C), 1 << 12)
    r.replay_window(b, _blocks_arr(first, pov, fl))
    got = r.replay_diffs(gf)
    lines = []
    for g in range(len(got)):
        dd = got.utxo_diff(g)
        for side, coll in (("add", dd.add), ("rem", dd.remove)):
            for (tid, idx), e in sorted(coll.items()):
                lines.append("%d %s %s %d %d %d %d %d %s" % (g, side, tid.hex(), idx, e["amount"], e["block_daa_score"], int(e["is_coinbase"]), e["spk_version"], e["script"].hex()))
    assert out.stdout.strip().splitlines() == lines
    assert len(lines) > 40
    r.close()
