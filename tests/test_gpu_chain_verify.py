"""kgv_replay_verify_chain on the GPU: verify_expected_utxo_state of every chain block of a replay window (commitment, accepted-id root,
coinbase rewards, the chain block's own transactions), against the reference's headers and blocks and against the CPU restatement
(oracle_chain.py) on mutated windows and on GHOSTDAG flags the fixtures do not carry."""
import copy
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle_body
import oracle_chain as oc
import pyref
from rusty_kaspa_b200 import Params
from rusty_kaspa_b200.muhash import MuHash, finalize_batch, prefix_combine
from rusty_kaspa_b200.replay import (CHAIN_HEADER_DTYPE, CHAIN_STATUS, MERGED_NON_DAA, MERGED_RED, REPLAY_ACCEPT_COINBASE, REPLAY_SKIP_SCRIPTS,
                                     REPLAY_VERIFY_ONLY, DagReplayer, replay_blocks_array)
from rusty_kaspa_b200.txbatch import build_batch
from rusty_kaspa_b200.validator import BodyRules, TxRules

pytestmark = pytest.mark.gpu

FIXTURES = ["simpa_goref_1060.json.gz", "simpa_goref_pruning_5000.json.gz"]
MAX_PAYLOAD_LEN, MAX_SPK_LEN = 204, 150
_plans = {}


def _plan(fixture):
    from golden_util import simpa_dag_replay_plan
    if fixture not in _plans:
        _plans[fixture] = simpa_dag_replay_plan(fixture)
    return _plans[fixture]


class Window:
    """One window of chain blocks: per chain block its mergeset in consensus order (the selected parent ACCEPT_COINBASE | SKIP_SCRIPTS),
    then its own body VERIFY_ONLY; headers from the fixture.  txs / flags may be mutated before replay()."""

    def __init__(self, fixture, chain_blocks):
        fx, by, order, sp, ordered_mergeset, chain = _plan(fixture)
        self.fx, self.genesis = fx, order[0]
        self.blocks, self.group_first, self.headers = [], [0], np.zeros(len(chain_blocks), dtype=CHAIN_HEADER_DTYPE)
        for g, b in enumerate(chain_blocks):
            s, ms = sp(b), ordered_mergeset(b)
            non_daa = len(ms) - (by[b]["daa_score"] - by[s]["daa_score"])
            for k, mb in enumerate(ms):
                self.blocks.append({"txs": copy.deepcopy(by[mb]["txs"]), "pov": by[b]["daa_score"], "flags": (REPLAY_ACCEPT_COINBASE | REPLAY_SKIP_SCRIPTS) if k == 0 else 0,
                                    "merged": MERGED_NON_DAA if (non_daa and mb == self.genesis) else 0, "hash": mb})
            self.blocks.append({"txs": copy.deepcopy(by[b]["txs"]), "pov": by[b]["daa_score"], "flags": REPLAY_VERIFY_ONLY, "merged": 0, "hash": b})
            self.group_first.append(len(self.blocks))
            h = self.headers[g]
            h["utxo_commitment"] = np.frombuffer(bytes.fromhex(by[b]["utxo_commitment"]), dtype=np.uint8)
            h["accepted_id_merkle_root"] = np.frombuffer(bytes.fromhex(by[b]["accepted_id_merkle_root"]), dtype=np.uint8)
            h["selected_parent_accepted_id_merkle_root"] = np.frombuffer(bytes.fromhex(by[s]["accepted_id_merkle_root"]), dtype=np.uint8)
            h["blue_score"], h["expected_subsidy"] = by[b]["blue_score"], oracle_body.SIMPA_SUBSIDY

    def merged_flags(self):
        return np.array([b["merged"] for b in self.blocks], dtype=np.uint8)

    def replay(self, r):
        txs, ranges = [], []
        for b in self.blocks:
            ranges.append((len(txs), len(b["txs"]), b["pov"], b["flags"]))
            txs.extend(b["txs"])
        self.first = [f for f, _, _, _ in ranges]
        self.batch, self.blocks_arr = build_batch(txs), replay_blocks_array(ranges)
        self.res, self.acc = r.replay_window(self.batch, self.blocks_arr, want_accept=True)
        return self


def _replayer(ctx, fixture):
    fx = _plan(fixture)[0]
    return DagReplayer(ctx, Params(coinbase_maturity=fx["coinbase_maturity"], storage_mass_parameter=fx["storage_mass_parameter"]), 1 << 16)


def _verify(r, w, init, headers=None):
    return r.verify_chain(w.group_first, w.headers if headers is None else headers, w.merged_flags(), init, TxRules(), BodyRules())


def restate(ctx, r, w, init, headers=None):
    """oracle_chain.verify_chain_block for every group of a replayed window: acceptance and fees from the window's results (the replay itself is
    checked against the CPU oracle elsewhere), commitments from the existing kgv_replay_muhash / prefix-combine / finalize-batch path"""
    headers = w.headers if headers is None else headers
    running = prefix_combine(ctx, r.replay_muhash(w.group_first), init)
    commits = finalize_batch(ctx, running)
    out, fees = [], []
    for g in range(len(w.group_first) - 1):
        b0, b1 = w.group_first[g], w.group_first[g + 1]
        merged = []
        for bi in range(b0, b1 - 1):
            f, n = w.first[bi], len(w.blocks[bi]["txs"])
            merged.append({"txs": w.blocks[bi]["txs"], "accepted": [bool(x) for x in w.acc[f:f + n]], "fees": [int(x) for x in w.res["fee"][f:f + n]],
                           "flags": w.blocks[bi]["merged"]})
        tail = w.blocks[b1 - 1]
        f = w.first[b1 - 1]
        ok = [int(s) == 0 for s in w.res["status"][f + 1:f + len(tail["txs"])]]
        h = headers[g]
        hd = {k: bytes(h[k]) for k in ("utxo_commitment", "accepted_id_merkle_root", "selected_parent_accepted_id_merkle_root")}
        hd["blue_score"], hd["expected_subsidy"] = int(h["blue_score"]), int(h["expected_subsidy"])
        o, bf = oc.verify_chain_block(merged, tail["txs"], ok, hd, commits[g].tobytes(), MAX_PAYLOAD_LEN, MAX_SPK_LEN)
        out.append(o)
        fees += bf + [0]
    return out, fees, running


def assert_equal_to_restatement(got, fees, exp, exp_fees):
    for g, (a, e) in enumerate(zip(got, exp)):
        assert int(a["status"]) == e["status"], (g, int(a["status"]), e["status"])
        assert (int(a["n_invalid_txs"]), int(a["n_txs"])) == (e["n_invalid_txs"], e["n_txs"]), g
        for k in ("utxo_commitment", "accepted_id_merkle_root", "coinbase_hash"):
            assert a[k].tobytes() == e[k], (g, k)
    for b, (a, e) in enumerate(zip(fees, exp_fees)):
        if e is not None:
            assert int(a) == e, b


@pytest.mark.parametrize("fixture", FIXTURES)
def test_whole_virtual_chain_verifies_and_matches_the_existing_path(gpu_ctx, fixture):
    chain = _plan(fixture)[5]
    w = Window(fixture, chain[1:])
    r = _replayer(gpu_ctx, fixture)
    w.replay(r)
    init = MuHash(gpu_ctx)
    got, fees, ms = _verify(r, w, init)
    bad = [g for g in range(len(got)) if got[g]["status"] != 0 or got[g]["n_invalid_txs"] != 0]
    assert not bad, (len(bad), bad[:5], got[bad[:5]] if bad else None)
    by = _plan(fixture)[1]
    for g, b in enumerate(chain[1:]):
        assert got[g]["utxo_commitment"].tobytes().hex() == by[b]["utxo_commitment"]
        assert got[g]["accepted_id_merkle_root"].tobytes().hex() == by[b]["accepted_id_merkle_root"]
        assert got[g]["n_txs"] == len(by[b]["txs"]) - 1
    # fees: the accepted non-coinbase transactions' fees of every merged block; multisets: the existing path's running values
    for bi, b in enumerate(w.blocks):
        f, n = w.first[bi], len(b["txs"])
        want = 0 if b["flags"] & REPLAY_VERIFY_ONLY else int(w.res["fee"][f + 1:f + n][w.acc[f + 1:f + n] == 1].sum())
        assert int(fees[bi]) == want, bi
    assert (ms == prefix_combine(gpu_ctx, r.replay_muhash(w.group_first))).all()
    if "1060" in fixture:  # the whole restatement, field by field
        exp, exp_fees, _ = restate(gpu_ctx, r, w, init)
        assert_equal_to_restatement(got, fees, exp, exp_fees)
    cbs = build_batch([by[b]["txs"][0] for b in chain[1:]])  # (staging another batch ends the window)
    assert (gpu_ctx.tx_hashes(cbs).reshape(-1, 32) == got["coinbase_hash"]).all()
    # the same chain in consecutive windows, each seeded with the previous one's last multiset: identical records
    r2 = _replayer(gpu_ctx, fixture)
    parts, at, init2 = [], 0, MuHash(gpu_ctx)
    step = (len(chain) - 1 + 2) // 3
    while at < len(chain) - 1:
        w2 = Window(fixture, chain[1 + at:1 + at + step]).replay(r2)
        g2, _, ms2 = _verify(r2, w2, init2)
        parts.append(g2)
        init2 = ms2[-1].tobytes()
        at += step
    assert (np.concatenate(parts) == got).all()
    r.close(); r2.close()


def _window_1060(ctx, n_chain=None):
    fixture = FIXTURES[0]
    chain = _plan(fixture)[5]
    w = Window(fixture, chain[1:] if n_chain is None else chain[1:1 + n_chain])
    r = _replayer(ctx, fixture)
    return w, r


def test_header_mutations_fail_exactly_their_chain_block(gpu_ctx):
    w, r = _window_1060(gpu_ctx)
    w.replay(r)
    init = MuHash(gpu_ctx)
    base, _, _ = _verify(r, w, init)
    assert (base["status"] == 0).all()
    rng = np.random.default_rng(11)
    for g in rng.choice(len(base), 6, replace=False):
        for field, status in (("utxo_commitment", 1), ("accepted_id_merkle_root", 2), ("selected_parent_accepted_id_merkle_root", 2),
                              ("expected_subsidy", 3), ("blue_score", 3)):
            h = w.headers.copy()
            if h.dtype[field].shape:
                h[g][field][int(rng.integers(32))] ^= 1 << int(rng.integers(8))
            else:
                h[g][field] += 1
            got, _, _ = _verify(r, w, init, h)
            assert got[g]["status"] == status, (g, field, got[g]["status"])
            others = np.arange(len(got)) != g
            assert (got["status"][others] == 0).all(), (g, field)
    r.close()


def _merge_group(w):
    """a group whose mergeset holds a block besides the selected parent"""
    for g in range(len(w.group_first) - 1):
        if w.group_first[g + 1] - w.group_first[g] - 1 >= 2:
            return g
    raise AssertionError("no group with a large enough mergeset")


def _set_payload_subsidy(tx, v):
    p = bytearray(tx["payload"])
    p[8:16] = (v & ((1 << 64) - 1)).to_bytes(8, "little")
    tx["payload"] = bytes(p)


BODY_MUTATIONS = ["subsidy+1", "subsidy-1", "subsidy-max", "payload-short", "out+1", "out-1", "swap", "extra-out", "drop-out", "mass", "extra-data",
                  "double-spend"]


@pytest.mark.parametrize("mutation", BODY_MUTATIONS)
def test_body_mutations_match_the_restatement(gpu_ctx, mutation):
    w, r = _window_1060(gpu_ctx)
    g = _merge_group(w) if mutation != "double-spend" else len(w.group_first) - 2  # the last chain block: everything before it is spent
    b0, bt = w.group_first[g], w.group_first[g + 1] - 1
    merged_cb = w.blocks[b0 + 1]["txs"][0]  # a non-selected merged block's coinbase
    chain_cb = w.blocks[bt]["txs"][0]       # the chain block's own coinbase (its VERIFY_ONLY copy)
    sub = int.from_bytes(merged_cb["payload"][8:16], "little")
    if mutation == "subsidy+1":
        _set_payload_subsidy(merged_cb, sub + 1)
    elif mutation == "subsidy-1":
        _set_payload_subsidy(merged_cb, sub - 1)
    elif mutation == "subsidy-max":
        _set_payload_subsidy(merged_cb, (1 << 64) - 1)  # with the selected parent's subsidy in the red sum: overflow
        w.blocks[b0]["merged"] = w.blocks[b0 + 1]["merged"] = MERGED_RED
    elif mutation == "payload-short":
        merged_cb["payload"] = merged_cb["payload"][:18]
    elif mutation in ("out+1", "out-1"):
        chain_cb["outputs"][0]["value"] += 1 if mutation == "out+1" else -1
    elif mutation == "swap":
        assert len(chain_cb["outputs"]) >= 2
        chain_cb["outputs"][0], chain_cb["outputs"][1] = chain_cb["outputs"][1], chain_cb["outputs"][0]
    elif mutation == "extra-out":
        chain_cb["outputs"].append(copy.deepcopy(chain_cb["outputs"][0]))
    elif mutation == "drop-out":
        chain_cb["outputs"].pop()
    elif mutation == "mass":
        chain_cb["mass"] = 1
    elif mutation == "extra-data":  # the miner data comes from this very payload: the block stays valid
        p = bytearray(chain_cb["payload"])
        if len(p) > 19 + p[18]:
            p[-1] ^= 0x55
        else:
            p.append(0x55)
        chain_cb["payload"] = bytes(p)
    elif mutation == "double-spend":  # a transaction an earlier group accepted: its inputs are spent by now
        src = [t for b in w.blocks[:bt] for t in b["txs"][1:]][-1]
        w.blocks[bt]["txs"].append(copy.deepcopy(src))
    w.replay(r)
    init = MuHash(gpu_ctx)
    got, fees, _ = _verify(r, w, init)
    exp, exp_fees, _ = restate(gpu_ctx, r, w, init)
    assert_equal_to_restatement(got, fees, exp, exp_fees)
    want = {"subsidy-max": CHAIN_STATUS["RewardOverflow"], "payload-short": CHAIN_STATUS["CoinbasePayloadUnparsable"], "extra-data": 0,
            "double-spend": 0}.get(mutation, CHAIN_STATUS["BadCoinbaseTransaction"])
    if mutation == "swap" and chain_cb["outputs"][0] == chain_cb["outputs"][1]:  # two equal rewards to one miner: the same transaction
        want = 0
    assert got[g]["status"] == want, (mutation, got[g])
    assert (np.delete(got["status"], g) == 0).all()
    if mutation == "double-spend":
        assert got[g]["n_invalid_txs"] == 1
    r.close()


def test_random_red_and_non_daa_flags_match_the_restatement(gpu_ctx):
    w, r = _window_1060(gpu_ctx)
    w.replay(r)
    init = MuHash(gpu_ctx)
    rng = np.random.default_rng(5)
    seen = set()
    for trial in range(4):
        for b in w.blocks:
            if not b["flags"] & REPLAY_VERIFY_ONLY:
                b["merged"] = int(rng.choice([0, 0, MERGED_RED, MERGED_NON_DAA, MERGED_RED | MERGED_NON_DAA]))
        got, fees, _ = _verify(r, w, init)
        exp, exp_fees, _ = restate(gpu_ctx, r, w, init)
        assert_equal_to_restatement(got, fees, exp, exp_fees)
        seen |= {int(s) for s in got["status"]}
    assert {0, CHAIN_STATUS["BadCoinbaseTransaction"]} <= seen
    r.close()


def test_host_and_device_pointers_and_call_order(gpu_ctx):
    import torch
    w, r = _window_1060(gpu_ctx, 40)
    w.replay(r)
    init = MuHash(gpu_ctx)
    host = _verify(r, w, init)
    # kgv_replay_muhash / kgv_replay_diffs before and after: the window stays current and the results do not change
    m1 = r.replay_muhash(w.group_first)
    d1 = r.replay_diffs(w.group_first)
    again = _verify(r, w, init)
    m2 = r.replay_muhash(w.group_first)
    d2 = r.replay_diffs(w.group_first)
    for a, b in zip(host, again):
        assert (a == b).all()
    assert (m1 == m2).all() and (d1.ranges == d2.ranges).all() and (d1.add_keys36 == d2.add_keys36).all()
    # device pointers
    lib, h = gpu_ctx._lib, gpu_ctx._h
    n_groups, nb = len(w.group_first) - 1, len(w.blocks)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    dh, dmf, dinit = dev(w.headers), dev(w.merged_flags()), dev(np.frombuffer(init.numerator + init.denominator, dtype=np.uint8))
    dres, dfee, dms = (torch.zeros(n, dtype=torch.uint8, device="cuda") for n in (n_groups * 112, nb * 8, n_groups * 768))
    torch.cuda.synchronize()
    gf = np.ascontiguousarray(w.group_first, dtype=np.uint32)
    rules, body = TxRules(), BodyRules()
    gpu_ctx._check(lib.kgv_replay_verify_chain(h, gf.ctypes.data, n_groups, dh.data_ptr(), dmf.data_ptr(), dinit.data_ptr(), ctypes.byref(rules),
                                               ctypes.byref(body), dres.data_ptr(), dfee.data_ptr(), dms.data_ptr()))
    torch.cuda.synchronize()
    assert dres.cpu().numpy().tobytes() == host[0].tobytes()
    assert dfee.cpu().numpy().tobytes() == host[1].tobytes() and dms.cpu().numpy().tobytes() == host[2].tobytes()
    # a mix of host and device pointers is refused
    assert lib.kgv_replay_verify_chain(h, gf.ctypes.data, n_groups, w.headers.ctypes.data, dmf.data_ptr(), dinit.data_ptr(), ctypes.byref(rules),
                                       ctypes.byref(body), dres.data_ptr(), None, None) != 0
    r.close()


def test_argument_errors(gpu_ctx):
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200._lib import KgvError
    w, r = _window_1060(gpu_ctx, 12)
    init = MuHash(gpu_ctx)
    # no window on a fresh context
    ctx2 = rk.GpuContext(0)
    try:
        gf = np.ascontiguousarray(w.group_first, dtype=np.uint32)
        res = np.zeros(len(gf) - 1, dtype=np.dtype((np.void, 112)))
        ib = np.frombuffer(init.numerator + init.denominator, dtype=np.uint8).copy()
        mf = w.merged_flags()
        rules, body = TxRules(), BodyRules()
        assert ctx2._lib.kgv_replay_verify_chain(ctx2._h, gf.ctypes.data, len(gf) - 1, w.headers.ctypes.data, mf.ctypes.data, ib.ctypes.data,
                                                 ctypes.byref(rules), ctypes.byref(body), res.ctypes.data, None, None) == -1
    finally:
        ctx2.close()
    w.replay(r)
    assert (_verify(r, w, init)[0]["status"] == 0).all()
    bad_groups = (list(w.group_first[:-1]) + [w.group_first[-1] - 1],   # does not tile
                  [0] + list(w.group_first[2:]))                          # a VERIFY_ONLY block inside a group
    for gf in bad_groups:
        with pytest.raises(KgvError):
            r.verify_chain(gf, w.headers[:len(gf) - 1], w.merged_flags()[:gf[-1]], init)  # arrays sized as the groups say: the call decides
    for bi, flags in ((w.group_first[1] - 1, 0), (w.group_first[1], 0)):  # a missing VERIFY_ONLY tail; a first block without ACCEPT_COINBASE
        w2 = Window(FIXTURES[0], _plan(FIXTURES[0])[5][1:13])
        w2.blocks[bi]["flags"] = flags
        w2.replay(r)
        with pytest.raises(KgvError):
            _verify(r, w2, init)
    # a window ended by another batch call
    w.replay(r)
    gpu_ctx.tx_ids(build_batch(w.blocks[0]["txs"]))
    with pytest.raises(KgvError):
        _verify(r, w, init)
    r.close()


def test_large_generated_windows_match_the_restatement(gpu_ctx):
    """Generated chains (simgen.FastDag, 150-transaction blocks) cut into groups of up to 41 blocks: over a thousand accepted ids in a group (the
    device-offset merkle path at depth) and mergesets past 32 blocks (the verdict kernel's multi-pass ballot, the 4-warp block stride).  Roots
    must equal merkle_hash(selected parent's root, calc_merkle_root(accepted ids)) recomputed on the host from accept and the tx ids,
    commitments the existing path's; the generated coinbase payloads are not in the reference's format, so every status is UNPARSABLE."""
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.replay import REPLAY_BLOCK_DTYPE
    g = simgen.FastDag(seed=41, n_keys=256, n_nonces=1024, coinbase_maturity=3, frac_invalid=0.02, coinbase_outputs=16)
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=3, storage_mass_parameter=g.C), 1 << 20)
    rng = np.random.default_rng(9)
    init = MuHash(gpu_ctx)
    max_ids = max_merged = 0
    for window in range(2):
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
        res, acc = r.replay_window(b, arr, want_accept=True)
        n_groups = len(gf) - 1
        headers = np.zeros(n_groups, dtype=CHAIN_HEADER_DTYPE)
        headers["selected_parent_accepted_id_merkle_root"] = rng.integers(0, 256, (n_groups, 32), dtype=np.uint8)
        mflags = rng.choice([0, 0, MERGED_RED, MERGED_NON_DAA], size=nb).astype(np.uint8)
        got, fees, ms = r.verify_chain(gf, headers, mflags, init)
        running = prefix_combine(gpu_ctx, r.replay_muhash(gf), init)
        assert (ms == running).all() and (got["utxo_commitment"] == finalize_batch(gpu_ctx, running)).all()
        assert (got["status"] == CHAIN_STATUS["CoinbasePayloadUnparsable"]).all()
        assert (b.txs["payload_len"][np.array(first[:-1])] < 19).all()  # the generator's coinbase payloads are below the minimum length
        for k in range(nb):
            lo, hi = first[k] + 1, first[k + 1]
            want = 0 if flags[k] & REPLAY_VERIFY_ONLY else int(res["fee"][lo:hi][acc[lo:hi] == 1].sum())
            assert int(fees[k]) == want, k
        ids = gpu_ctx.tx_ids(b)  # (staging another batch ends the window)
        for gi in range(n_groups):
            b0, bt = gf[gi], gf[gi + 1] - 1
            sel = [first[b0]] + [t for k in range(b0, bt) for t in range(first[k] + 1, first[k + 1]) if acc[t]]
            root = pyref.blake2b_keyed(b"MerkleBranchHash", headers[gi]["selected_parent_accepted_id_merkle_root"].tobytes()
                                       + pyref.merkle_root([ids[t].tobytes() for t in sel]))
            assert got[gi]["accepted_id_merkle_root"].tobytes() == root, (window, gi)
            lo, hi = first[bt] + 1, first[bt + 1]
            assert (int(got[gi]["n_invalid_txs"]), int(got[gi]["n_txs"])) == (int((res["status"][lo:hi] != 0).sum()), hi - lo)
            max_ids, max_merged = max(max_ids, len(sel)), max(max_merged, bt - b0)
        init = MuHash(gpu_ctx, ms[-1, :384].tobytes(), ms[-1, 384:].tobytes())
    assert max_ids > 1024 and max_merged > 32, (max_ids, max_merged)  # a tree of 11 levels or more; the ballot's second pass
    r.close(); g.close()


def test_cpp_mirror_prints_the_same_verdicts(gpu_ctx, tmp_path):
    """kgv::TransactionValidator::verify_chain_blocks (include/kgv.hpp, driven by tests/cpp/chain_verify_mirror_test.cpp) on fixture 1 with one
    chain block's coinbase output changed: the same records, fees and last multiset as the Python binding"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe, libdir = str(tmp_path / "chain_verify_mirror_test"), os.path.join(root, "rusty_kaspa_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(root, "tests", "cpp", "chain_verify_mirror_test.cpp"), "-L" + libdir, "-l:libkgv.so",
                    "-Wl,-rpath," + libdir], check=True)
    w, r = _window_1060(gpu_ctx, 40)
    g = _merge_group(w)
    w.blocks[w.group_first[g + 1] - 1]["txs"][0]["outputs"][0]["value"] += 1
    w.replay(r)
    init = MuHash(gpu_ctx)
    got, fees, ms = _verify(r, w, init)
    assert got[g]["status"] == CHAIN_STATUS["BadCoinbaseTransaction"] and (np.delete(got["status"], g) == 0).all()
    d = str(tmp_path)
    for name, arr in (("txs", w.batch.txs), ("inputs", w.batch.inputs), ("outputs", w.batch.outputs), ("arena", w.batch.arena), ("blocks", w.blocks_arr),
                      ("groups", np.array(w.group_first, np.uint32)), ("headers", w.headers), ("merged", w.merged_flags()),
                      ("init", np.frombuffer(init.numerator + init.denominator, dtype=np.uint8))):
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    fx = w.fx
    out = subprocess.run([exe, d, str(fx["coinbase_maturity"]), str(fx["storage_mass_parameter"])], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.strip().splitlines()
    want = ["%d %d %d %s %s %s" % (x["status"], x["n_invalid_txs"], x["n_txs"], x["utxo_commitment"].tobytes().hex(), x["accepted_id_merkle_root"].tobytes().hex(),
                                   x["coinbase_hash"].tobytes().hex()) for x in got]
    assert lines[:len(got)] == want
    assert lines[len(got)] == " ".join(str(int(f)) for f in fees) and lines[len(got) + 1] == ms[-1].tobytes().hex()
    assert lines[len(got) + 2] == "threw"
    r.close()


def test_mirror_refuses_arrays_that_do_not_cover_the_window(gpu_ctx):
    w, r = _window_1060(gpu_ctx, 6)
    w.replay(r)
    init = MuHash(gpu_ctx)
    with pytest.raises(ValueError):
        r.verify_chain(w.group_first, w.headers, w.merged_flags()[:-1], init)
    with pytest.raises(ValueError):
        r.verify_chain(w.group_first, w.headers[:-1], w.merged_flags(), init)
    assert (_verify(r, w, init)[0]["status"] == 0).all()
    r.close()
