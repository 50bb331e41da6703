"""kgv_validate_block_bodies against the CPU restatement of the reference's body rules (oracle_body.py), field by field: the two DAG
fixtures, the reference's example block with its mutations, every status and every ordered pair of violated rules, the edges of the mass
and payload rules, per-block lock-time contexts, and the linear set checks at sizes and block counts the pairwise kernel could not take."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
import oracle_body as ob  # noqa: E402
import oracle_isolation as oi  # noqa: E402

pytestmark = pytest.mark.gpu
U64 = (1 << 64) - 1
MAX_BLOCK_MASS, MAX_PAYLOAD = 500_000, 204
SPK = bytes([0x20]) + bytes(range(32)) + bytes([0xAC])


def processor(ctx, max_block_mass=MAX_BLOCK_MASS, **rule_overrides):
    from rusty_kaspa_b200.validator import BlockBodyProcessor, BodyRules, TxRules
    return BlockBodyProcessor(ctx, TxRules(**rule_overrides), BodyRules(max_block_mass, MAX_PAYLOAD))


def layout(blocks):
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import block_headers
    first = np.cumsum([0] + [len(b["transactions"]) for b in blocks]).astype(np.uint32)
    h = block_headers(blocks, 0)
    h["expected_subsidy"] = [b["expected_subsidy"] for b in blocks]
    h["past_median_time"] = [b.get("past_median_time", 0) for b in blocks]
    return build_batch([t for b in blocks for t in b["transactions"]]), first, h


def check(ctx, blocks, max_block_mass=MAX_BLOCK_MASS, isolation_only=False, roots=True, **rule_overrides):
    """one call for all blocks; every field of every verdict, the masses and the roots equal the oracle's.  Returns the statuses."""
    p = processor(ctx, max_block_mass, **rule_overrides)
    batch, first, h = layout(blocks)
    res, masses, got_roots = p.validate_bodies(batch, first, h, isolation_only)
    rules = dict(oi.mainnet_rules(), **rule_overrides)
    exp = ob.ok_validate_bodies(blocks, rules, max_block_mass, MAX_PAYLOAD, isolation_only)
    for k, (verdict, m) in enumerate(exp):
        got = {f: int(res[k][f]) for f in verdict}
        assert got == verdict, (k, ob.NAME.get(got["status"]), got, ob.NAME[verdict["status"]], verdict)
        assert tuple(int(x) for x in masses[k]) == m, k
        if roots:
            assert got_roots[k].tobytes() == ob.calc_hash_merkle_root(blocks[k]["transactions"]), k
    return [v["status"] for v, _ in exp]


# ---- generated blocks: valid by construction, no signatures needed by any body rule
def coinbase(blue_score, subsidy=50, script=SPK):
    return {"version": 0, "inputs": [], "outputs": [{"value": subsidy, "spk_version": 0, "script": SPK}], "lock_time": 0, "subnetwork_id": oi.COINBASE,
            "gas": 0, "payload": ob.coinbase_payload(blue_score, subsidy, script), "mass": 0}


def spend(rng, n_in=2, n_out=2, mass=10):
    return {"version": 0, "lock_time": 0, "subnetwork_id": oi.NATIVE, "gas": 0, "payload": b"", "mass": mass,
            "inputs": [{"txid": rng.bytes(32), "index": int(rng.integers(0, 4)), "sigscript": rng.bytes(66), "sequence": 0, "sig_op_count": 1} for _ in range(n_in)],
            "outputs": [{"value": int(rng.integers(1, 10**9)), "spk_version": 0, "script": SPK} for _ in range(n_out)]}


def seal(block):
    block["hash_merkle_root"] = ob.calc_hash_merkle_root(block["transactions"])
    return block


def make_block(rng, n_txs=4, blue_score=7, daa_score=1000, subsidy=50, **tx_kw):
    return seal({"transactions": [coinbase(blue_score, subsidy)] + [spend(rng, **tx_kw) for _ in range(n_txs - 1)], "daa_score": daa_score,
                 "blue_score": blue_score, "past_median_time": 1_700_000_000_000, "expected_subsidy": subsidy})


# ---- the reference's data
@pytest.mark.parametrize("name,n", [("simpa_goref_1060.json.gz", 266), ("simpa_goref_pruning_5000.json.gz", 5001)])
def test_dag_fixture_in_one_call(gpu_ctx, name, n):
    """every block of a reference DAG with its real header: all Ok, masses equal, computed roots equal to the headers'"""
    blocks = ob.fixture_blocks(name)
    assert len(blocks) == n
    assert set(check(gpu_ctx, blocks, isolation_only=True)) == {0}
    assert set(check(gpu_ctx, blocks[1:])) == {0}  # the context stage without the genesis, which the reference stores without validating
    _, _, roots = processor(gpu_ctx).validate_bodies(*layout(blocks))
    assert all(roots[k].tobytes() == b["hash_merkle_root"] for k, b in enumerate(blocks))


def test_reference_example_block_and_mutations(gpu_ctx):
    """validate_body_in_isolation_test: the example block and its eight mutations in one call, then one block per call"""
    cases = ob.reference_example_blocks()
    blocks = [c[1] for c in cases]
    assert check(gpu_ctx, blocks, isolation_only=True) == [ob.STATUS[c[2]] for c in cases]
    p = processor(gpu_ctx)
    for name, block, err in cases:
        res, masses = p.validate_body_in_isolation(block)
        assert ob.NAME[int(res["status"])] == err, name
        assert (int(masses["compute_mass"]) > 0) == (err == "Ok")


# ---- every status, and the earlier rule wins
def _violate(rule, b, rng):
    t = b["transactions"]
    if rule == 2:
        b["bad_root"] = True
    elif rule == "3a":
        t[0]["subnetwork_id"] = oi.NATIVE
    elif rule == "3b":
        t[2]["subnetwork_id"] = oi.COINBASE
    elif rule == 4:
        t[1]["gas"] = 1
    elif rule in ("5c", "5t", "5s"):
        pass  # by the mass limit of the call, see below
    elif rule == "6a":
        t.append(copy.deepcopy(t[1]))
    elif rule == "6b":
        t[3]["inputs"][0]["txid"], t[3]["inputs"][0]["index"] = t[1]["inputs"][1]["txid"], t[1]["inputs"][1]["index"]
    elif rule == "6c":
        b["chain"] = True
    elif rule == "7a":
        t[0]["payload"] = t[0]["payload"][:10]
    elif rule == "7b":
        b["blue_score"] += 1
    elif rule == "7c":
        b["expected_subsidy"] += 1
    elif rule == 8:
        t[2]["lock_time"] = b["daa_score"]


RULES = [2, "3a", "3b", 4, "5s", "6a", "6b", "6c", "7a", "7b", "7c", 8]
RULE_STATUS = {2: 2, "3a": 3, "3b": 4, 4: 5, "5s": 8, "6a": 9, "6b": 10, "6c": 11, "7a": 12, "7b": 13, "7c": 14, 8: 15}


def _violating_block(rng, rules):
    import pyref
    b = make_block(rng, 5)
    if "5s" in rules:
        b["transactions"][3]["mass"] = MAX_BLOCK_MASS  # with the other commitments the running total passes the limit at tx 3
    for r in rules:
        _violate(r, b, rng)
    if b.pop("chain", False):  # after every other change to transaction 1
        t = b["transactions"]
        t[3]["inputs"][1]["txid"], t[3]["inputs"][1]["index"] = pyref.tx_id(t[1]), 1
    seal(b)
    if b.pop("bad_root", False):
        b["hash_merkle_root"] = bytes(31) + b"\x01"
    return b


def test_every_status_and_every_ordered_pair(gpu_ctx):
    rng = np.random.default_rng(11)
    blocks = [make_block(rng, 5), dict(make_block(rng, 1), transactions=[], hash_merkle_root=bytes(32))]
    want = [0, 1]
    for r in RULES:
        blocks.append(_violating_block(rng, [r]))
        want.append(RULE_STATUS[r])
    for i, early in enumerate(RULES):
        for late in RULES[i + 1:]:
            if {early, late} == {"3a", "3b"} or {early, late} == {"6a", "6c"}:
                continue  # one changes what the other's transaction is
            blocks.append(_violating_block(rng, [late, early]))
            want.append(RULE_STATUS[early])
    got = check(gpu_ctx, blocks)
    assert got == want
    assert set(got) >= set(range(16)) - {6, 7}  # compute / transient excess: test_mass_edges
    # the isolation stage alone stops after the set checks
    iso = check(gpu_ctx, blocks, isolation_only=True)
    assert iso == [s if s < 12 else 0 for s in want]


def test_mass_edges(gpu_ctx):
    rng = np.random.default_rng(5)
    rules = oi.mainnet_rules()
    base = make_block(rng, 6, mass=0)
    for t in base["transactions"]:
        for x in t["inputs"]:
            x["sig_op_count"] = 0  # without signature operations the transient mass (4 per byte) is the largest of the three
    seal(base)
    per_tx = [oi.ok_tx_non_contextual_masses(t, rules) for t in base["transactions"]]
    compute, transient = sum(c for c, _ in per_tx), sum(t for _, t in per_tx)
    assert transient > compute
    # total == limit passes, limit + 1 fails in the last tx (transient is the larger sum here)
    assert check(gpu_ctx, [base], max_block_mass=transient) == [0]
    assert check(gpu_ctx, [base], max_block_mass=transient - 1) == [7]
    # compute before transient before storage when several pass at one tx
    both = copy.deepcopy(base)
    both["transactions"][2]["mass"] = compute  # storage passes any limit below `compute` at tx 2 already
    seal(both)
    lim = per_tx[1][0] + per_tx[2][0] - 1      # compute passes at tx 2 as well (and transient, four times the size, too)
    assert check(gpu_ctx, [both], max_block_mass=lim) == [6]
    two = copy.deepcopy(base)
    lim = per_tx[1][1] + per_tx[2][1] - 1      # transient passes at tx 2, compute does not
    two["transactions"][2]["mass"] = lim + 1   # and so does storage
    seal(two)
    assert check(gpu_ctx, [two], max_block_mass=lim) == [7]
    only_storage = copy.deepcopy(base)
    only_storage["transactions"][5]["mass"] = transient + 1
    seal(only_storage)
    assert check(gpu_ctx, [only_storage], max_block_mass=transient) == [8]
    # commitments that saturate at u64::MAX, against a limit of u64::MAX (passes) and below it (fails at the tx where the sum saturates)
    sat = copy.deepcopy(base)
    sat["transactions"][2]["mass"] = U64 - 5
    sat["transactions"][4]["mass"] = 1 << 63
    seal(sat)
    assert check(gpu_ctx, [sat], max_block_mass=U64) == [0]
    assert check(gpu_ctx, [sat], max_block_mass=U64 - 1) == [8]
    # a body longer than one scan chunk whose first excess is in its last tx, beside bodies that pass
    long = make_block(rng, 300, n_in=1, n_out=1, mass=1)
    long["transactions"][-1]["mass"] = 10**7
    seal(long)
    tot = max(sum(oi.ok_tx_non_contextual_masses(t, rules)[k] for t in long["transactions"]) for k in (0, 1))
    assert check(gpu_ctx, [base, long, base], max_block_mass=tot) == [0, 8, 0]


def test_payload_edges(gpu_ctx):
    rng = np.random.default_rng(6)
    blocks = []
    full = ob.coinbase_payload(7, 50, bytes(150), extra=bytes(40))
    for n in range(0, ob.MIN_PAYLOAD_LENGTH + 150 + 2):  # every length: too short, cannot hold its script, exact, with extra data
        b = make_block(rng, 2)
        b["transactions"][0]["payload"] = full[:n]
        blocks.append(seal(b))
    for spk_len in (149, 150, 151, 255):                   # the length byte at and above the maximum, in a payload long enough for it
        b = make_block(rng, 2)
        b["transactions"][0]["payload"] = ob.coinbase_payload(7, 50)[:18] + bytes([spk_len]) + bytes(185)
        blocks.append(seal(b))
    b = make_block(rng, 2)
    b["transactions"][0]["payload"] = bytes(205)           # above max_coinbase_payload_len
    blocks.append(seal(b))
    got = check(gpu_ctx, blocks)
    assert got[:19] == [12] * 19 and got[19 + 150] == 0 and got[19 + 149] == 12 and got[-1] == 12 and got[-2] == 12 and got[-4] == 0


def test_lock_time_uses_each_blocks_own_context(gpu_ctx):
    rng = np.random.default_rng(7)
    blocks = []
    for daa, pmt, lock in [(1000, 5 * 10**11 + 50, 1000), (1001, 5 * 10**11 + 50, 1000), (1000, 5 * 10**11 + 50, 5 * 10**11 + 50),
                           (1000, 5 * 10**11 + 51, 5 * 10**11 + 50), (999, 5 * 10**11, 1000)]:
        b = make_block(rng, 40, daa_score=daa)
        b["past_median_time"] = pmt
        b["transactions"][37]["lock_time"] = lock
        b["transactions"][37]["inputs"][0]["sequence"] = U64  # the second input decides
        blocks.append(seal(b))
    assert check(gpu_ctx, blocks) == [15, 0, 15, 0, 15]


# ---- the set checks in linear work
def test_repeats_whose_first_offender_is_not_in_the_first_group(gpu_ctx):
    """two repeated outpoints and two repeated ids: the reference reports the repeat that comes first in iteration order, not the one whose
    first occurrence comes first"""
    rng = np.random.default_rng(8)
    b = make_block(rng, 12, n_in=3)
    t = b["transactions"]
    t[9]["inputs"][2] = dict(t[1]["inputs"][0])   # group A: first seen early, repeated late
    t[6]["inputs"][0] = dict(t[5]["inputs"][1])   # group B: first seen later, repeated earlier -> the offender
    seal(b)
    b2 = make_block(rng, 12)
    b2["transactions"] += [copy.deepcopy(b2["transactions"][8]), copy.deepcopy(b2["transactions"][2])]
    seal(b2)
    batch, first, h = layout([b, b2])
    res, _, _ = processor(gpu_ctx).validate_bodies(batch, first, h)
    assert (int(res[0]["status"]), int(res[0]["index"])) == (10, 5 * 3 + 0)
    assert (int(res[1]["status"]), int(res[1]["index"])) == (9, 12 + 12)
    check(gpu_ctx, [b, b2])


def test_large_bodies_against_the_oracle_and_the_set_checks(gpu_ctx):
    """a body of 50 000 inputs and one of 5 000 transactions (their sets live in device memory, not shared memory), each with a late repeat"""
    rng = np.random.default_rng(9)
    wide = make_block(rng, 51, n_in=1000, n_out=1)
    wide["transactions"][44]["inputs"][700] = dict(wide["transactions"][3]["inputs"][10])
    many = make_block(rng, 5000, n_in=1, n_out=1)
    many["transactions"].append(copy.deepcopy(many["transactions"][4321]))
    small = make_block(rng, 3)
    blocks = [seal(wide), small, seal(many)]
    assert check(gpu_ctx, blocks, max_block_mass=U64) == [10, 0, 9]
    batch, first, h = layout(blocks)
    sets = gpu_ctx.block_set_checks(batch, first)
    res, _, _ = processor(gpu_ctx, U64).validate_bodies(batch, first, h)
    assert sets["status"].tolist() == [2, 0, 1] and sets["index"].tolist() == res["index"].tolist()
    assert int(sets[0]["index"]) == 43 * 1000 + 700 and int(sets[2]["index"]) == 51 + 3 + 5000


def _utxo_key_hash(txid, index):
    """key_hash of kgv_utxo.cuh, the unkeyed hash the UTXO table places outpoints by"""
    w = [int.from_bytes(txid[8 * k:8 * k + 8], "little") for k in range(4)]
    h = w[0] ^ (w[1] * 0x9E3779B97F4A7C15 & U64) ^ (w[2] * 0xC2B2AE3D27D4EB4F & U64) ^ (w[3] * 0x165667B19E3779F9 & U64) ^ (index * 0xD6E8FEB86659FD93 & U64)
    h ^= h >> 29
    h = h * 0xBF58476D1CE4E5B9 & U64
    return h ^ (h >> 32)


def test_outpoints_crafted_to_share_one_public_hash(gpu_ctx):
    """a peer chooses the outpoints of a body: 50 000 distinct ones built so that the UTXO table's public key_hash is one value for all of
    them, with a repeat placed late.  The sets place items by a hash keyed with a secret salt, so the verdict is the oracle's and the call
    takes the time of a body of random outpoints, not a quadratic walk along one probe run"""
    import time
    rng = np.random.default_rng(13)
    honest = make_block(rng, 51, n_in=1000, n_out=1)
    crafted = copy.deepcopy(honest)
    target = 0x0123456789ABCDEF
    for t in crafted["transactions"][1:]:
        for x in t["inputs"]:
            tail = rng.bytes(24)
            w = [int.from_bytes(tail[8 * k:8 * k + 8], "little") for k in range(3)]
            w0 = target ^ (w[0] * 0x9E3779B97F4A7C15 & U64) ^ (w[1] * 0xC2B2AE3D27D4EB4F & U64) ^ (w[2] * 0x165667B19E3779F9 & U64) ^ (x["index"] * 0xD6E8FEB86659FD93 & U64)
            x["txid"] = w0.to_bytes(8, "little") + tail
    ins = [x for t in crafted["transactions"] for x in t["inputs"]]
    assert len({_utxo_key_hash(x["txid"], x["index"]) for x in ins}) == 1 and len({(x["txid"], x["index"]) for x in ins}) == 50_000
    for b in (honest, crafted):
        b["transactions"][48]["inputs"][999] = dict(b["transactions"][2]["inputs"][5])
        seal(b)
    assert check(gpu_ctx, [crafted, honest], max_block_mass=U64) == [10, 10]
    p = processor(gpu_ctx, U64)
    ms = []
    for b in (honest, crafted):
        args = layout([b])
        p.validate_bodies(*args)
        t0 = time.perf_counter()
        res, _, _ = p.validate_bodies(*args)
        ms.append((time.perf_counter() - t0) * 1e3)
        assert (int(res[0]["status"]), int(res[0]["index"])) == (10, 47 * 1000 + 999)
    assert ms[1] < 5 * ms[0] + 50, ms


def test_many_tiny_bodies_with_repeats(gpu_ctx):
    """3 000 bodies of 2 to 4 transactions of one input: sets of 4 to 8 and 2 to 6 slots, where most probe walks meet an occupied slot and
    many start at the last slot and continue at slot 0; a third of the bodies repeat an outpoint or a transaction"""
    rng = np.random.default_rng(14)
    blocks = []
    for k in range(3000):
        b = make_block(rng, int(rng.integers(2, 5)), n_in=1, n_out=1)
        t = b["transactions"]
        if k % 3 == 1 and len(t) > 2:
            t[-1]["inputs"][0] = dict(t[1]["inputs"][0])
        elif k % 3 == 2:
            t.append(copy.deepcopy(t[-1]))
        blocks.append(seal(b))
    got = check(gpu_ctx, blocks, roots=False)
    assert set(got) == {0, 9, 10}


def test_equal_to_block_set_checks_on_many_random_blocks(gpu_ctx):
    """10 000 small random bodies with outpoints drawn from a small pool, more than 65 535 bodies in one call, empty bodies between full ones:
    the body verdict's set-check part is kgv_block_set_checks' answer"""
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import BLOCK_HEADER_CTX_DTYPE
    rng = np.random.default_rng(10)
    pool = [(rng.bytes(32), k) for k in range(64)]
    txs, first = [], [0]
    for k in range(10_000):
        cb = coinbase(7)
        blk = [cb]
        for _ in range(int(rng.integers(0, 6))):
            t = spend(rng, n_in=int(rng.integers(1, 4)))
            for x in t["inputs"]:
                if rng.random() < 0.2:
                    x["txid"], x["index"] = pool[int(rng.integers(0, 64))]
            blk.append(t)
        if len(blk) > 2 and rng.random() < 0.05:
            blk.append(copy.deepcopy(blk[1]))
        txs += blk
        first.append(len(txs))
    for k in range(60_000):  # single-coinbase bodies and empty ones: 70 000 bodies in all
        if k % 3:
            txs.append(coinbase(7))
        first.append(len(txs))
    batch = build_batch(txs)
    first = np.array(first, dtype=np.uint32)
    n = len(first) - 1
    assert n > 65535
    h = np.zeros(n, dtype=BLOCK_HEADER_CTX_DTYPE)
    h["hash_merkle_root"] = gpu_ctx.block_hash_merkle_roots(batch, first)
    h["blue_score"], h["expected_subsidy"], h["daa_score"] = 7, 50, 1000
    sets = gpu_ctx.block_set_checks(batch, first)
    res, masses, roots = processor(gpu_ctx).validate_bodies(batch, first, h)
    empty = np.diff(first) == 0
    assert (res["status"][empty] == 1).all() and (roots[empty] == 0).all() and (sets["status"][empty] == 0).all()
    same_tx = res["status"] == 5  # both draws of one transaction hit one pool entry: TxDuplicateInputs comes before the block's double spend
    assert (res["tx_status"][same_tx] == 27).all() and (sets["status"][same_tx] != 0).all() and same_tx.sum() < 1000
    full = ~empty & ~same_tx
    assert (res["status"][full] == np.where(sets["status"][full] == 0, 0, sets["status"][full] + 8)).all()
    assert (res["index"][full] == sets["index"][full]).all()
    assert {0, 1, 2}.issubset(set(sets["status"].tolist())) and (masses["storage_mass"][res["status"] != 0] == 0).all()
    # a sample of them against the oracle as well
    blocks = [{"transactions": txs[first[k]:first[k + 1]], "hash_merkle_root": h[k]["hash_merkle_root"].tobytes(), "daa_score": 1000, "blue_score": 7,
               "past_median_time": 0, "expected_subsidy": 50} for k in range(0, 10_000, 97)]
    check(gpu_ctx, blocks, roots=False)


def test_host_and_device_pointers_give_the_same_bytes(gpu_ctx):
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    rng = np.random.default_rng(12)
    blocks = [make_block(rng, 5)] + [_violating_block(rng, [r]) for r in RULES] + [dict(make_block(rng, 1), transactions=[], hash_merkle_root=bytes(32))]
    p = processor(gpu_ctx)
    batch, first, h = layout(blocks)
    res, masses, roots = p.validate_bodies(batch, first, h)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    t = {k: dev(getattr(batch, k)) for k in ("txs", "inputs", "outputs", "arena")}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(batch.txs), t["inputs"].data_ptr(), len(batch.inputs), t["outputs"].data_ptr(), len(batch.outputs), None,
                     t["arena"].data_ptr(), len(batch.arena))
    n = len(blocks)
    dh = dev(h)
    out = [torch.zeros(n * w, dtype=torch.uint8, device="cuda") for w in (32, 24, 32)]
    torch.cuda.synchronize()
    gpu_ctx._check(gpu_ctx._lib.kgv_validate_block_bodies(gpu_ctx._h, ctypes.byref(cb), first.ctypes.data, n, dh.data_ptr(), ctypes.byref(p.rules),
                                                          ctypes.byref(p.body_rules), 0, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr()))
    gpu_ctx.synchronize()
    for got, want in zip(out, (res, masses, roots)):
        assert got.cpu().numpy().tobytes() == want.tobytes()
    # a mix of host and device pointers is refused
    rc = gpu_ctx._lib.kgv_validate_block_bodies(gpu_ctx._h, ctypes.byref(cb), first.ctypes.data, n, h.ctypes.data, ctypes.byref(p.rules),
                                                ctypes.byref(p.body_rules), 0, out[0].data_ptr(), None, None)
    assert rc != 0
