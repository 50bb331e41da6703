"""kgv_validate_mempool_txs (validate_mempool_transaction_in_utxo_context, utxo_validation.rs:341-397) against the CPU oracle.

The expected outcome of every transaction is composed from the oracle in the reference's order: populate (the caller's entries first, the
rest from the oracle's UTXO state, every input tried) -> MissingTxOutpoints -> oracle storage mass (MassIncomputable) -> the oracle's populated
validation with SkipMassCheck (maturity, amounts, sequence lock, scripts) -> the feerate threshold in Python floats (IEEE f64 as Rust's
`as f64` and `/`), which comes before the scripts."""
import ctypes
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import oracle_tx
from rusty_kaspa_b200 import GpuUtxoSet, KgvError, Params, TransactionValidator
from rusty_kaspa_b200.simgen import SUBNET_NATIVE, SimDag, entries_to_arrays, funded_window, tx_id
from rusty_kaspa_b200.txbatch import ENTRY_DTYPE, build_batch

pytestmark = pytest.mark.gpu

U64MAX = 2**64 - 1  # UNACCEPTED_DAA_SCORE of an entry created by an in-mempool parent
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _key36(i):
    return bytes(i["txid"]) + int(i["index"]).to_bytes(4, "little")


def _batch(txs, supplied):
    """the batch and its `supplied` mask: supplied[ti][k] is an entry dict (the caller's) or None (look it up)"""
    b = build_batch(txs, supplied)
    mask = np.array([e is not None for es in supplied for e in es], dtype=bool)
    return b, mask


def oracle_mempool(ora, ost, txs, supplied, pov, op, thresholds=None, nc_mass=None):
    """expected (results, masses, final entries: dict or None per input)"""
    n = len(txs)
    res = np.zeros(n, dtype=oracle_tx.RESULT_DTYPE)
    mass = np.zeros(n, dtype=np.uint64)
    finals = []
    per_tx = []
    for t, sup in zip(txs, supplied):
        f = [s if s is not None else ost.get(_key36(i)) for i, s in zip(t["inputs"], sup)]
        finals.extend(f)
        per_tx.append(f)
    pb = build_batch(txs, [[e if e is not None else {"amount": 0, "spk_version": 0, "script": b""} for e in f] for f in per_tx])
    for ti, f in enumerate(per_tx):
        r = res[ti]
        if any(e is None for e in f):
            r["status"] = 1
            continue
        m = oracle_tx.storage_mass(ora, pb, ti, op.storage_mass_parameter)
        if m is None:
            r["status"] = 6
            continue
        mass[ti] = m
        e = oracle_tx.validate_populated(ora, pb, ti, pov, 2, op)  # SkipMassCheck
        r["status"], r["script_err"], r["fail_input"], r["fee"] = e["status"], e["script_err"], e["fail_input"], e["fee"]
        if e["status"] in (2, 3, 4, 5, 8):
            continue
        thr = None if thresholds is None else float(thresholds[ti])
        if thr is not None and not math.isnan(thr):
            div = max(int(m), int(nc_mass[ti]))
            assert div > 0
            if float(int(e["fee"])) / float(div) <= thr:
                r["status"], r["script_err"], r["fail_input"] = 13, 0, 0
    return res, mass, finals


def same(got, exp, what=""):
    gr, gm, ge, ga = got
    er, em, ef = exp
    assert (gr["status"] == er["status"]).all(), (what, np.nonzero(gr["status"] != er["status"])[0][:8], gr["status"][:20], er["status"][:20])
    assert (gr["script_err"] == er["script_err"]).all(), what
    bad = (gr["status"] == 2)
    assert (gr["fail_input"][bad] == er["fail_input"][bad]).all(), what
    feeful = ~np.isin(gr["status"], (1, 2, 3, 4, 5, 6, 12))
    assert (gr["fee"][feeful] == er["fee"][feeful]).all(), what
    assert (gm == em).all(), (what, np.nonzero(gm != em)[0][:8])
    assert len(ge) == len(ef)
    for i, (g, e) in enumerate(zip(ge, ef)):
        if e is None:
            assert g["pad_"][0] == 1 and g["amount"] == 0 and g["script_len"] == 0, (what, i)
            continue
        assert g["pad_"][0] == 0, (what, i)
        assert int(g["amount"]) == e["amount"] and int(g["block_daa_score"]) == e.get("block_daa_score", 0), (what, i)
        assert int(g["spk_version"]) == e["spk_version"] and bool(g["is_coinbase"]) == bool(e.get("is_coinbase", False)), (what, i)
        assert bytes(ga[int(g["script_off"]):int(g["script_off"]) + int(g["script_len"])]) == bytes(e["script"]), (what, i)


class Pool:
    """a virtual UTXO set (GPU table and oracle state) and three unapplied blocks whose transactions form a mempool with chains"""

    def __init__(self, gpu_ctx, oracle, seed=23):
        self.dag = dag = SimDag(seed=seed, n_keys=64, n_nonces=128, mix=(0.5, 0.2, 0.15, 0.15), frac_invalid=0.0, coinbase_maturity=4, coinbase_outputs=10)
        self.op = oracle_tx.params(coinbase_maturity=4, storage_mass_parameter=dag.C)
        self.params = Params(coinbase_maturity=4, storage_mass_parameter=dag.C)
        self.tv = TransactionValidator(gpu_ctx, self.params)
        self.us = GpuUtxoSet(gpu_ctx, 1 << 14)
        self.ost = oracle_tx.State(oracle)
        self.ora = oracle
        self.last_coinbase = None
        for _ in range(12):
            txs, pov = dag.make_block(20)
            b = build_batch(txs)
            acc = np.ones(len(txs), dtype=np.uint8)
            assert self.ost.accept(b, acc, pov) == 0
            self.ost.commit()
            self.us.add_transactions(b, acc, pov)
            self.last_coinbase = txs[0]
        # mempool: parents (block A), children (B) and grandchildren (C) - never applied to the set
        self.layers = []
        dag.frac_invalid = 0.15
        for _ in range(3):
            txs, pov = dag.make_block(60)
            self.layers.append(txs[1:])
        self.pov = pov
        self.pool = [t for layer in self.layers for t in layer]
        self.outputs = {}  # outpoint -> the entry an in-mempool parent's output gives (UNACCEPTED_DAA_SCORE)
        for t in self.pool:
            tid = tx_id(t)
            for k, o in enumerate(t["outputs"]):
                self.outputs[tid + k.to_bytes(4, "little")] = {"amount": o["value"], "spk_version": o["spk_version"], "script": o["script"],
                                                               "block_daa_score": U64MAX, "is_coinbase": False}

    def ok_parents(self):
        """the parents (not chained) the oracle accepts"""
        txs = self.layers[0]
        r, _, _ = oracle_mempool(self.ora, self.ost, txs, [[None] * len(t["inputs"]) for t in txs], self.pov, self.op)
        return [t for t, s in zip(txs, r["status"]) if s == 0]

    def supplied(self, txs):
        return [[self.outputs.get(_key36(i)) for i in t["inputs"]] for t in txs]

    def run(self, txs, supplied, thresholds=None, nc_mass=None, tv=None, op=None):
        b, mask = _batch(txs, supplied)
        got = (tv or self.tv).validate_mempool_transactions_in_utxo_context(self.us, b, self.pov, thresholds, nc_mass, supplied=mask)
        exp = oracle_mempool(self.ora, self.ost, txs, supplied, self.pov, op or self.op, thresholds, nc_mass)
        return got, exp

    def close(self):
        self.us.close()
        self.ost.close()


@pytest.fixture
def pool(gpu_ctx, oracle):
    p = Pool(gpu_ctx, oracle)
    yield p
    p.close()


def test_chained_mempool_batch(pool):
    """parents, children and grandchildren with the in-mempool parents' outputs supplied as u64::MAX-score entries: verdicts, fees, masses
    and returned entries equal the oracle's; the same batch without the caller's entries leaves the chained ones MissingTxOutpoints"""
    sup = pool.supplied(pool.pool)
    n_chained = sum(e is not None for es in sup for e in es)
    children = {tx_id(t) for t in pool.layers[1]}
    grandchildren = [t for t in pool.layers[2] if any(bytes(i["txid"]) in children for i in t["inputs"])]
    assert n_chained > 30 and grandchildren
    got, exp = pool.run(pool.pool, sup)
    same(got, exp, "chained")
    st = set(int(s) for s in got[0]["status"])
    assert 0 in st and 1 in st and (9 in st or 10 in st), st
    ok = got[0]["status"] == 0
    chained_ok = [ti for ti, es in enumerate(sup) if ok[ti] and any(e is not None for e in es)]
    assert len(chained_ok) > 10
    assert ok.sum() > 60 and (got[0]["fee"][ok] == 1).all()
    # the mirror of the block path (kgv_validate_txs) calls every chained transaction an orphan
    old = pool.tv.validate_mempool_transactions_in_parallel(pool.us, build_batch(pool.pool), pool.pov)
    assert (old["status"][chained_ok] == 1).all()
    nothing = [[None] * len(t["inputs"]) for t in pool.pool]
    got2, exp2 = pool.run(pool.pool, nothing)
    same(got2, exp2, "no caller entries")
    assert (got2[0]["status"][chained_ok] == 1).all()


def test_supplied_looked_up_or_mixed_agree(pool):
    """a batch whose inputs all exist in the set: every entry supplied, none, or every other one - identical results"""
    txs = pool.layers[0]
    table = [[pool.ost.get(_key36(i)) for i in t["inputs"]] for t in txs]
    modes = {"all": table, "none": [[None] * len(es) for es in table],
             "mixed": [[e if (ti + k) % 2 else None for k, e in enumerate(es)] for ti, es in enumerate(table)]}
    outs = {}
    for name, sup in modes.items():
        got, exp = pool.run(txs, sup)
        same(got, exp, name)
        outs[name] = got
    for name in ("none", "mixed"):
        a, b = outs["all"], outs[name]
        assert (a[0] == b[0]).all() and (a[1] == b[1]).all(), name
        for x, y in zip(a[2], b[2]):
            assert x["amount"] == y["amount"] and x["pad_"][0] == y["pad_"][0]


def test_caller_entry_wins_and_partial_populate(pool):
    """an entry the caller supplies for an outpoint the set also holds wins (the fee shows it); partially missing inputs give
    MissingTxOutpoints and the inputs that were found still come back filled"""
    t0 = next(t for t in pool.ok_parents() if len(t["inputs"]) == 2)
    real = [pool.ost.get(_key36(i)) for i in t0["inputs"]]
    changed = dict(real[0], amount=real[0]["amount"] + 1000)
    got, exp = pool.run([t0, t0], [[None, None], [changed, None]])
    same(got, exp, "caller wins")
    assert got[0]["fee"][1] == got[0]["fee"][0] + 1000 and got[2][2]["amount"] == changed["amount"]
    orphan = {**t0, "inputs": [dict(t0["inputs"][0]), dict(t0["inputs"][1], txid=bytes(range(32)))]}
    got, exp = pool.run([orphan], [[None, None]])
    same(got, exp, "partial")
    assert got[0]["status"][0] == 1 and got[2][0]["pad_"][0] == 0 and got[2][0]["amount"] == real[0]["amount"] and got[2][1]["pad_"][0] == 1


def test_mass_is_computed_not_checked(pool):
    """a wrong committed mass is no error and the computed mass is returned; a transaction both mass-incomputable and spending an immature
    coinbase output gives MassIncomputable here (the mass comes first) and ImmatureCoinbaseSpend through kgv_validate_txs"""
    t0 = pool.ok_parents()[0]
    wrong = dict(t0, mass=t0["mass"] + 7)
    cb_id = tx_id(pool.last_coinbase)
    immature = {"version": 0, "inputs": [{"txid": cb_id, "index": 0, "sigscript": b"", "sequence": 0, "sig_op_count": 1}],
                "outputs": [{"value": 0, "spk_version": 0, "script": b"\x51"}], "lock_time": 0, "subnetwork_id": SUBNET_NATIVE, "gas": 0,
                "payload": b"", "mass": 0}
    got, exp = pool.run([t0, wrong, immature], [[None] * len(t0["inputs"]), [None] * len(t0["inputs"]), [None]])
    same(got, exp, "mass")
    assert got[0]["status"][1] == got[0]["status"][0] == 0 and got[1][1] == got[1][0] != wrong["mass"]
    assert got[0]["status"][2] == 6
    blk = pool.tv.validate_transactions_in_parallel(pool.us, build_batch([t0, wrong, immature]), pool.pov)
    assert list(blk["status"]) == [got[0]["status"][0], 7, 2]


def test_sequence_lock_on_unaccepted_entries(pool):
    """check_sequence_lock on a u64::MAX-score entry: (i64)u64::MAX + lock - 1 >= pov, i.e. a relative lock of pov + 2 blocks, pov + 1 passes"""
    child = next(t for t in pool.layers[1] if all(pool.outputs.get(_key36(i)) for i in t["inputs"]))
    sup = pool.supplied([child])[0]
    cases = []
    for lock in (pool.pov, pool.pov + 1, pool.pov + 2, pool.pov + 3, 0xFFFFFFFF):
        c = dict(child, inputs=[dict(i, sequence=lock) for i in child["inputs"]])
        cases.append(c)
    got, exp = pool.run(cases, [sup] * len(cases))
    same(got, exp, "sequence")
    assert list(got[0]["status"][:2] != 8) == [True, True] and list(got[0]["status"][2:] == 8) == [True, True, True]


def test_feerate_threshold(pool):
    """fee / max(storage mass, non-contextual mass) <= threshold is FeerateTooLow: equality fails, one sompi more passes, NaN checks
    nothing; with fee and divisor above 2^53 the u64 -> f64 rounding decides; a zero divisor is a caller error"""
    t0 = next(t for t in pool.ok_parents() if len(t["inputs"]) == 1)
    ent = pool.ost.get(_key36(t0["inputs"][0]))
    base, _ = pool.run([t0], [[None]])
    assert base[0]["status"][0] == 0
    m = int(base[1][0])
    more = dict(t0, outputs=[dict(t0["outputs"][0], value=t0["outputs"][0]["value"] - 1)] + t0["outputs"][1:])  # fee 2 (signature now wrong)
    nc = 300
    div = max(m, nc)
    eq = 1.0 / float(div)
    tiny = dict(t0, outputs=[dict(o, value=1) for o in t0["outputs"]])  # outputs of 1 sompi: a storage mass of about 2 C
    big_fee = 2**60 + 127                     # rounds to 2^60 as f64
    big = dict(ent, amount=len(t0["outputs"]) + big_fee)
    m_big = int(oracle_mempool(pool.ora, pool.ost, [tiny], [[big]], pool.pov, pool.op)[1][0])
    assert m_big > 0  # with an input this large the storage mass is the divisor unless the caller's mass is larger
    exact_vs_f64 = Fraction(big_fee, 2**54) <= Fraction(64.0)
    assert not exact_vs_f64 and float(big_fee) / float(2**54) <= 64.0  # exact arithmetic would let it through, f64 does not
    up_fee = dict(ent, amount=len(t0["outputs"]) + 2**60 + 129)
    exact_fee = dict(ent, amount=len(t0["outputs"]) + 2**60)
    rz = lambda x: float(x >> (x.bit_length() - 53) << (x.bit_length() - 53))  # truncating u64 -> f64
    assert float(2**60 + 129) > 64.0 * 2**54 and rz(2**60 + 129) / float(2**54) == 64.0
    assert float(2**60) / float(2**54 + 3) <= math.nextafter(64.0, 0.0) < float(2**60) / rz(2**54 + 3)
    rows = [  # (tx, supplied entry, threshold, non-contextual mass)
        (t0, None, float("nan"), 0),
        (t0, None, eq, nc),
        (t0, None, math.nextafter(eq, 0.0), nc),
        (more, None, eq, nc),
        (tiny, big, float(big_fee) / float(m_big), 0),
        (tiny, big, 64.0, 2**54),
        (tiny, big, math.nextafter(64.0, 0.0), 2**54),
        (tiny, big, 64.0, 2**54 + 1),           # divisor rounds to 2^54 too
        (tiny, big, float(big_fee) / float(2**55 + 3), 2**55 + 3),
        # rows that only round-to-nearest passes (truncating conversions or division would give the other verdict):
        (t0, None, 0.2, 5),                                  # 1 / 5 rounds UP to 0.2000000000000000111 = float 0.2: equal
        (t0, None, math.nextafter(0.2, 0.0), 5),             # the truncated quotient would equal this threshold
        (tiny, up_fee, 64.0, 2**54),                         # fee 2^60 + 129 rounds up to 2^60 + 256: quotient just above 64
        (tiny, exact_fee, math.nextafter(64.0, 0.0), 2**54 + 3),  # divisor rounds up to 2^54 + 4: quotient 64 - 2^-46
    ]
    txs = [r[0] for r in rows]
    sup = [[r[1]] for r in rows]
    thr = np.array([r[2] for r in rows])
    ncm = np.array([r[3] for r in rows], dtype=np.uint64)
    got, exp = pool.run(txs, sup, thr, ncm)
    same(got, exp, "feerate")
    assert list(got[0]["status"]) == [0, 13, 0, 9, 13, 13, 9, 13, 13, 13, 0, 9, 13], list(got[0]["status"])
    # NULL args: no thresholds at all
    got_none, _ = pool.run(txs, sup)
    assert (got_none[0]["status"] != 13).all()
    # max(storage mass, non-contextual mass) == 0 with a threshold: the reference asserts, the call refuses
    tv0 = TransactionValidator(pool.tv.ctx, Params(coinbase_maturity=4, storage_mass_parameter=0))
    b, mask = _batch([t0], [[None]])
    with pytest.raises(KgvError):
        tv0.validate_mempool_transactions_in_utxo_context(pool.us, b, pool.pov, np.array([0.5]), np.array([0], dtype=np.uint64), supplied=mask)
    r0 = tv0.validate_mempool_transactions_in_utxo_context(pool.us, b, pool.pov, np.array([0.5]), np.array([5], dtype=np.uint64), supplied=mask)
    assert r0[1][0] == 0 and r0[0]["status"][0] == 13  # fee 1 / 5 <= 0.5


def test_sigcache_sees_only_transactions_that_reach_scripts(pool):
    """with a SigCache attached, FeerateTooLow and context-failed transactions make no lookups or inserts: the counters equal those of
    validating just the transactions that reached the scripts"""
    from rusty_kaspa_b200.validator import SigCache
    txs = pool.pool
    sup = pool.supplied(txs)
    rng = np.random.default_rng(5)
    thr = np.where(rng.random(len(txs)) < 0.3, 1.0, np.nan)  # fee 1 / mass <= 1: FeerateTooLow
    ncm = np.full(len(txs), 1, dtype=np.uint64)
    got, exp = pool.run(txs, sup, thr, ncm)
    same(got, exp, "uncached")
    res = got[0]
    reached = [ti for ti in range(len(txs)) if res["status"][ti] in (0, 9, 10)]
    assert (res["status"] == 13).sum() > 20 and len(reached) > 40 and (res["status"] == 1).any()
    ctx = pool.tv.ctx
    sc = SigCache(ctx, 1 << 16)
    sc.attach()
    try:
        b, mask = _batch(txs, sup)
        again = pool.tv.validate_mempool_transactions_in_utxo_context(pool.us, b, pool.pov, thr, ncm, supplied=mask)
        assert (again[0] == res).all()
        c_mempool = sc.counters()
        sc.clear()
        c0 = sc.counters()
        entries = got[2]
        per_tx, k = [], 0
        for t in txs:
            per_tx.append(entries[k:k + len(t["inputs"])]); k += len(t["inputs"])
        sub = [txs[ti] for ti in reached]
        sub_ents = []
        for ti in reached:
            row = []
            for e in per_tx[ti]:
                o = int(e["script_off"])
                row.append({"amount": int(e["amount"]), "spk_version": int(e["spk_version"]), "script": bytes(got[3][o:o + int(e["script_len"])]),
                            "block_daa_score": int(e["block_daa_score"]), "is_coinbase": bool(e["is_coinbase"])})
            sub_ents.append(row)
        pool.tv.validate_populated_transactions(build_batch(sub, sub_ents), pool.pov, flags=2)
        c_sub = sc.counters()
        assert c_mempool["lookups"] == c_sub["lookups"] - c0["lookups"] > 0, (c_mempool, c_sub, c0)
        assert c_mempool["inserts"] == c_sub["inserts"] - c0["inserts"] > 0, (c_mempool, c_sub, c0)
    finally:
        sc.close()


def test_nonstandard_scripts_with_caller_entries(gpu_ctx, oracle):
    """non-standard spends whose entries the caller supplies (or the set holds) are decided by the host script engine inside the call"""
    from rusty_kaspa_b200.validator import script_execute
    from test_gpu_host_vm import _custom_spends
    from test_host_vm import oracle_verdicts
    txs, ents = _custom_spends(64, seed=11)
    us = GpuUtxoSet(gpu_ctx, 1 << 12)
    keys = np.frombuffer(b"".join(_key36(t["inputs"][0]) for t in txs[1::2]), dtype=np.uint8).reshape(-1, 36)
    arr, arena = entries_to_arrays([ents[ti][0] for ti in range(1, len(txs), 2)])
    us.apply_diff(add_keys36=keys, add_entries=arr, add_bytes=arena)
    sup = [[ents[ti][0]] if ti % 2 == 0 else [None] for ti in range(len(txs))]
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=0, storage_mass_parameter=0))
    b, mask = _batch(txs, sup)
    res, mass, fin, arena = tv.validate_mempool_transactions_in_utxo_context(us, b, 1000, supplied=mask)
    full = build_batch(txs, ents)
    verdicts = oracle_verdicts(oracle, full)
    names = set()
    for i in range(len(txs)):
        exp = script_execute(full, i, 0, verdicts)
        got = 0 if res[i]["status"] == 0 else int(res[i]["script_err"])
        assert res[i]["status"] in (0, 9) and got == exp, (i, res[i], exp)
        names.add(got)
    assert 0 in names and len(names) >= 3
    assert (fin["pad_"][:, 0] == 0).all() and (fin["amount"] == 10**9).all() and (fin["block_daa_score"] == 5).all()
    for ti, e in enumerate(fin):  # supplied (even ti) and looked-up (odd ti) scripts, returned although the host engine ran after populate
        assert bytes(arena[int(e["script_off"]):int(e["script_off"]) + int(e["script_len"])]) == ents[ti][0]["script"], ti
    us.close()


def _device_call(gpu_ctx, us, b, mask, pov, params, thr, ncm):
    """the same call with every array in device memory (the call returns without synchronising)"""
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    from rusty_kaspa_b200.validator import MEMPOOL_ARGS_DTYPE, RESULT_DTYPE
    ent = b.entries.copy()
    ent["pad_"][:, 0] = np.where(mask, 0, 1)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    args = np.zeros(len(b.txs), dtype=MEMPOOL_ARGS_DTYPE)
    args["feerate_threshold"], args["non_contextual_mass"] = thr, ncm
    t = {k: dev(v) for k, v in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", ent), ("arena", b.arena), ("args", args))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(b.txs), t["inputs"].data_ptr(), len(b.inputs), t["outputs"].data_ptr(), len(b.outputs),
                     t["entries"].data_ptr(), t["arena"].data_ptr(), len(b.arena))
    n, ni = len(b.txs), len(b.inputs)
    res = torch.zeros(n * 16, dtype=torch.uint8, device="cuda")
    mass = torch.zeros(n * 8, dtype=torch.uint8, device="cuda")
    eo = torch.zeros(ni * 32, dtype=torch.uint8, device="cuda")
    cap = len(b.arena) + 128 * ni
    so = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    used = ctypes.c_size_t()
    gpu_ctx._check(gpu_ctx._lib.kgv_validate_mempool_txs(gpu_ctx._h, us._h, ctypes.byref(cb), pov, ctypes.byref(params), t["args"].data_ptr(), res.data_ptr(),
                                                         mass.data_ptr(), eo.data_ptr(), so.data_ptr(), cap, ctypes.byref(used)))
    gpu_ctx._check(gpu_ctx._lib.kgv_synchronize(gpu_ctx._h))
    return (res.cpu().numpy().view(RESULT_DTYPE), mass.cpu().numpy().view(np.uint64), eo.cpu().numpy().view(ENTRY_DTYPE), so.cpu().numpy()[:used.value])


def test_host_and_device_pointers_and_sizes(pool, gpu_ctx):
    """host and device pointers give the same bytes; batches of 1, 16 and 256 transactions; a too small script buffer is reported with
    the size it needs, before any signature is verified"""
    txs = (pool.pool * 2)[:256]  # the pool repeated: each transaction is validated on its own
    assert len(txs) == 256
    sup = pool.supplied(txs)
    thr = np.where(np.arange(len(txs)) % 4 == 0, 1.0, np.nan)
    ncm = np.full(len(txs), 1, dtype=np.uint64)
    for n in (1, 16, 256):
        got, exp = pool.run(txs[:n], sup[:n], thr[:n], ncm[:n])
        same(got, exp, "n=%d" % n)
    b, mask = _batch(txs, sup)
    host = pool.tv.validate_mempool_transactions_in_utxo_context(pool.us, b, pool.pov, thr, ncm, supplied=mask)
    devr = _device_call(gpu_ctx, pool.us, b, mask, pool.pov, pool.params, thr, ncm)
    for h, d in zip(host, devr):
        assert h.tobytes() == d.tobytes()
    from rusty_kaspa_b200.verifier import _c_batch
    from rusty_kaspa_b200.txbatch import TxBatch
    ent = b.entries.copy()
    ent["pad_"][:, 0] = np.where(mask, 0, 1)
    cb = _c_batch(TxBatch(b.txs, b.inputs, b.outputs, ent, b.arena))
    res = np.zeros(len(txs), dtype=oracle_tx.RESULT_DTYPE)
    mass = np.zeros(len(txs), dtype=np.uint64)
    eo = np.zeros(len(b.inputs), dtype=ENTRY_DTYPE)
    small = np.zeros(8, dtype=np.uint8)
    used = ctypes.c_size_t()
    rc = gpu_ctx._lib.kgv_validate_mempool_txs(gpu_ctx._h, pool.us._h, ctypes.byref(cb), pool.pov, ctypes.byref(pool.params), None, res.ctypes.data,
                                               mass.ctypes.data, eo.ctypes.data, small.ctypes.data, len(small), ctypes.byref(used))
    assert rc == -3 and used.value == len(host[3])
    import torch
    dargs = torch.zeros(16 * len(txs), dtype=torch.uint8, device="cuda")  # device args beside host outputs: refused, nothing dereferenced
    rc = gpu_ctx._lib.kgv_validate_mempool_txs(gpu_ctx._h, pool.us._h, ctypes.byref(cb), pool.pov, ctypes.byref(pool.params), dargs.data_ptr(), res.ctypes.data,
                                               mass.ctypes.data, None, None, 0, None)
    assert rc == -1


def test_large_batch_through_the_key_cache(gpu_ctx, oracle):
    """3 x 10^4 transactions over 64 keys: more Schnorr items than the verify grid has threads, so the launch deduplicates keys and reads
    key records; half of the entries supplied, half looked up"""
    fk, fe, txs = funded_window(30_000, n_keys=64, n_nonces=256, mix=(0.6, 0.1, 0.3, 0.0))
    ents, k = [], 0
    for t in txs:
        ents.append(list(fe[k:k + len(t["inputs"])])); k += len(t["inputs"])
    for ti in range(0, len(txs), 97):  # a few bad signatures
        ss = txs[ti]["inputs"][0]["sigscript"]
        txs[ti]["inputs"][0]["sigscript"] = ss[:20] + bytes([ss[20] ^ 2]) + ss[21:]
    us = GpuUtxoSet(gpu_ctx, 1 << 17)
    table_keys = [_key36(i) for ti, t in enumerate(txs) if ti % 2 for i in t["inputs"]]
    table_ents = [e for ti, es in enumerate(ents) if ti % 2 for e in es]
    arr, arena = entries_to_arrays(table_ents)
    us.apply_diff(add_keys36=np.frombuffer(b"".join(table_keys), dtype=np.uint8).reshape(-1, 36), add_entries=arr, add_bytes=arena)
    sup = [es if ti % 2 == 0 else [None] * len(es) for ti, es in enumerate(ents)]
    from rusty_kaspa_b200.simgen import DEFAULT_STORAGE_MASS_PARAMETER as C
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=100, storage_mass_parameter=C))
    b, mask = _batch(txs, sup)
    got = tv.validate_mempool_transactions_in_utxo_context(us, b, 10, supplied=mask)
    form = gpu_ctx.debug_key_form(False)["form"]
    assert form in ("plain", "comb"), form
    # expected: every entry is known here (the table half is exactly what was inserted), so the oracle validates the populated batch
    res_e = np.zeros(len(txs), dtype=oracle_tx.RESULT_DTYPE)
    mass_e = np.zeros(len(txs), dtype=np.uint64)
    full = build_batch(txs, ents)
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=C)
    for ti in range(len(txs)):
        m = oracle_tx.storage_mass(oracle, full, ti, C)
        mass_e[ti] = m
        e = oracle_tx.validate_populated(oracle, full, ti, 10, 2, op)
        res_e[ti] = e
    same(got, (res_e, mass_e, [e for es in ents for e in es]), "10k")
    assert (got[0]["status"] == 0).sum() > 29000 and (got[0]["status"] == 9).any()
    us.close()


def test_cpp_mirror(pool, tmp_path):
    """TransactionValidator::validate_mempool_transactions_in_utxo_context of include/kgv.hpp on the chained batch, with thresholds"""
    binary = str(tmp_path / "mempool_mirror_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", binary, os.path.join(HERE, "cpp", "mempool_mirror_test.cpp"), "-L" + os.path.join(ROOT, "rusty_kaspa_b200"),
                    "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    txs = pool.pool
    sup = pool.supplied(txs)
    thr = np.where(np.arange(len(txs)) % 3 == 0, 1.0, np.nan)
    ncm = np.full(len(txs), 1, dtype=np.uint64)
    b, mask = _batch(txs, sup)
    ent = b.entries.copy()
    ent["pad_"][:, 0] = np.where(mask, 0, 1)
    d = str(tmp_path)
    for name, arr in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", ent), ("arena", b.arena)):
        arr.tofile(os.path.join(d, name + ".bin"))
    from rusty_kaspa_b200.validator import MEMPOOL_ARGS_DTYPE
    args = np.zeros(len(txs), dtype=MEMPOOL_ARGS_DTYPE)
    args["feerate_threshold"], args["non_contextual_mass"] = thr, ncm
    args.tofile(os.path.join(d, "args.bin"))
    keys, fents, farena = pool.us.export()
    keys.tofile(os.path.join(d, "fund_keys.bin")); fents.tofile(os.path.join(d, "fund_entries.bin")); farena.tofile(os.path.join(d, "fund_arena.bin"))
    out = subprocess.run([binary, d, str(pool.pov), str(pool.dag.C)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.split("\n")
    tx_lines = [l.split() for l in lines if l.startswith("tx ")]
    in_lines = [l.split() for l in lines if l.startswith("in ")]
    er, em, ef = oracle_mempool(pool.ora, pool.ost, txs, sup, pool.pov, pool.op, thr, ncm)
    assert len(tx_lines) == len(txs) and len(in_lines) == len(b.inputs)
    for ti, f in enumerate(tx_lines):
        st = int(f[1])
        assert st == er["status"][ti] and int(f[2]) == er["script_err"][ti] and int(f[5]) == em[ti], (ti, f, er[ti], em[ti])
        if st in (0, 8, 9, 10, 13):
            assert int(f[4]) == er["fee"][ti]
    assert (er["status"] == 13).any()
    for f, e in zip(in_lines, ef):
        if e is None:
            assert f[1] == "0"
            continue
        assert f[1] == "1" and int(f[2]) == e["amount"] and int(f[3]) == e.get("block_daa_score", 0)
        assert (f[6] if f[6] != "-" else "") == bytes(e["script"]).hex()
