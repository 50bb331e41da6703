"""kgv_validate_txs_in_isolation and kgv_validate_mempool_txs_in_parallel against the CPU restatement (oracle_isolation.py) and the
reference's own cases.

The mempool expectation is composed in the reference's order (validate_mempool_transaction_impl, processor.rs:823-839): the oracle's
isolation -> finality verdict, and for the transactions that pass both, the UTXO-context expectation of test_gpu_mempool's oracle fed with
the oracle's non-contextual masses."""
import ctypes

import numpy as np
import pytest

import oracle_isolation as oi
from rusty_kaspa_b200.txbatch import ENTRY_DTYPE, build_batch
from rusty_kaspa_b200.validator import RESULT_DTYPE, TX_MASSES_DTYPE, SigCache, TxRules
from test_gpu_mempool import Pool, _batch, _key36, oracle_mempool, same

pytestmark = pytest.mark.gpu

U64 = 2**64 - 1
DAA, PMT = 400_000_000_000, 600_000_000_000  # on either side of LOCK_TIME_THRESHOLD
SMALL = dict(max_tx_inputs=40, max_tx_outputs=40, max_signature_script_len=300, max_script_public_key_len=60, mass_per_tx_byte=1,
             mass_per_script_pub_key_byte=10, mass_per_sig_op=1000, ghostdag_k=10, coinbase_payload_script_public_key_max_len=30)
INDEXED = (16, 18, 22, 23, 24, 31)


def _iso(tv, txs, rules, daa=DAA, pmt=PMT, finality=True):
    return tv.validate_txs_in_isolation(build_batch(txs), TxRules(**rules), daa, pmt, finality)


def _expect(txs, rules, daa=DAA, pmt=PMT, finality=True):
    st = np.array([oi.ok_tx_validate(t, rules, daa, pmt, finality) for t in txs], dtype=np.uint64)
    ms = np.array([oi.ok_tx_non_contextual_masses(t, rules) for t in txs], dtype=np.uint64).reshape(-1, 2)
    return st, ms


def _agree(got, txs, rules, what, **kw):
    res, masses = got
    st, ms = _expect(txs, rules, **kw)
    bad = np.nonzero(res["status"] != st[:, 0])[0]
    assert len(bad) == 0, (what, [(int(i), int(res["status"][i]), int(st[i, 0])) for i in bad[:8]])
    ix = np.isin(res["status"], INDEXED)
    assert (res["fail_input"][ix] == st[ix, 1]).all(), what
    assert (res["fail_input"][~ix] == 0).all() and (res["fee"] == 0).all() and (res["script_err"] == 0).all(), what
    assert (masses["compute_mass"] == ms[:, 0]).all() and (masses["transient_mass"] == ms[:, 1]).all(), what
    return res


@pytest.fixture
def tv(gpu_ctx):
    from rusty_kaspa_b200 import TransactionValidator
    return TransactionValidator(gpu_ctx)


def _device_iso(gpu_ctx, txs, rules, daa, pmt, finality=True):
    """kgv_validate_txs_in_isolation with every array in device memory"""
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    b = build_batch(txs)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    t = {k: dev(v) for k, v in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("arena", b.arena))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(b.txs), t["inputs"].data_ptr(), len(b.inputs), t["outputs"].data_ptr(), len(b.outputs), None,
                     t["arena"].data_ptr(), len(b.arena))
    res = torch.zeros(len(txs) * 16, dtype=torch.uint8, device="cuda")
    ms = torch.zeros(len(txs) * 16, dtype=torch.uint8, device="cuda")
    gpu_ctx._check(gpu_ctx._lib.kgv_validate_txs_in_isolation(gpu_ctx._h, ctypes.byref(cb), ctypes.byref(TxRules(**rules)), daa, pmt, 0 if finality else 1,
                                                              res.data_ptr(), ms.data_ptr()))
    gpu_ctx._check(gpu_ctx._lib.kgv_synchronize(gpu_ctx._h))
    return res.cpu().numpy().view(RESULT_DTYPE), ms.cpu().numpy().view(TX_MASSES_DTYPE)


def test_reference_cases_host_and_device(tv, gpu_ctx):
    """validate_tx_in_isolation_test's transactions and the NotFinalized cases: the reference's error class and index, host and device pointers"""
    cases, rules = oi.isolation_golden_cases()
    fin = oi.finality_golden_cases(DAA, PMT)
    txs = [c[1] for c in cases] + [c[1] for c in fin]
    exp = [oi.STATUS[c[2]] for c in cases] + [oi.STATUS[c[2]] for c in fin]
    got = _agree(_iso(tv, txs, rules), txs, rules, "golden")
    assert list(got["status"]) == exp
    dres, dms = _device_iso(gpu_ctx, txs, rules, DAA, PMT)
    hres, hms = _iso(tv, txs, rules)
    assert dres.tobytes() == hres.tobytes() and dms.tobytes() == hms.tobytes()
    # plain validate_tx_in_isolation: the finality cases all pass
    skip = _iso(tv, txs, rules, finality=False)[0]
    assert (skip["status"][len(cases):] == 0).all()


def _base(rng, n_in=None, n_out=None):
    n_in = int(rng.integers(1, 6)) if n_in is None else n_in
    n_out = int(rng.integers(1, 5)) if n_out is None else n_out
    return {"version": 0, "lock_time": 0, "subnetwork_id": oi.NATIVE, "gas": 0, "payload": rng.bytes(int(rng.integers(0, 20))), "mass": 0,
            "inputs": [{"txid": rng.bytes(32), "index": int(rng.integers(0, 2**32)), "sigscript": rng.bytes(int(rng.integers(0, 120))),
                        "sequence": (U64, 0, int(rng.integers(0, 2**63)))[int(rng.integers(0, 3))], "sig_op_count": int(rng.integers(0, 4))} for _ in range(n_in)],
            "outputs": [{"value": int(rng.integers(1, 10**12)), "spk_version": 0, "script": rng.bytes(int(rng.integers(0, 40)))} for _ in range(n_out)]}


def _mutants(rng, r):
    """one rule at a time, with the boundary values on both sides"""
    M = oi.MAX_SOMPI
    T = oi.LOCK_TIME_THRESHOLD
    cbk = oi.COINBASE

    def coinbase(n_out, spk=5, mass=0, inputs=0):
        t = _base(rng, inputs or 1, n_out)
        t.update(subnetwork_id=cbk, mass=mass, inputs=t["inputs"][:inputs])
        for o in t["outputs"]:
            o["script"] = bytes(spk)
        return t

    def with_(t, **kw):
        t.update(kw)
        return t

    def at(t, kind, i, **kw):
        t[kind][i].update(kw)
        return t

    gens = [
        lambda: _base(rng),
        lambda: with_(_base(rng), inputs=[]),
        lambda: _base(rng, n_in=r["max_tx_inputs"]),
        lambda: _base(rng, n_in=r["max_tx_inputs"] + 1),
        lambda: at(_base(rng, n_in=4), "inputs", int(rng.integers(0, 4)), sigscript=bytes(r["max_signature_script_len"])),
        lambda: at(_base(rng, n_in=4), "inputs", int(rng.integers(0, 4)), sigscript=bytes(r["max_signature_script_len"] + 1)),
        lambda: _base(rng, n_out=r["max_tx_outputs"]),
        lambda: _base(rng, n_out=r["max_tx_outputs"] + 1),
        lambda: at(_base(rng, n_out=4), "outputs", int(rng.integers(0, 4)), script=bytes(r["max_script_public_key_len"])),
        lambda: at(_base(rng, n_out=4), "outputs", int(rng.integers(0, 4)), script=bytes(r["max_script_public_key_len"] + 1)),
        lambda: coinbase(r["ghostdag_k"] + 2),
        lambda: coinbase(r["ghostdag_k"] + 3),
        lambda: coinbase(2, mass=1),
        lambda: coinbase(2, inputs=1),
        lambda: coinbase(3, spk=r["coinbase_payload_script_public_key_max_len"]),
        lambda: at(coinbase(3, spk=r["coinbase_payload_script_public_key_max_len"]), "outputs", 1,
                   script=bytes(r["coinbase_payload_script_public_key_max_len"] + 1)),
        lambda: at(_base(rng, n_out=3), "outputs", 2, value=0),
        lambda: at(_base(rng, n_out=3), "outputs", int(rng.integers(0, 3)), value=M + 1),
        lambda: with_(_base(rng, n_out=2), outputs=[{"value": M - 7, "spk_version": 0, "script": b""}, {"value": 7, "spk_version": 0, "script": b""}]),
        lambda: with_(_base(rng, n_out=2), outputs=[{"value": M - 7, "spk_version": 0, "script": b""}, {"value": 8, "spk_version": 0, "script": b""}]),
        lambda: with_(_base(rng), outputs=[{"value": M, "spk_version": 0, "script": b""} for _ in range(40)]),  # the u64 sum would wrap
        lambda: with_(_base(rng), outputs=[{"value": 1, "spk_version": 0, "script": b""}] * 35 + [{"value": M, "spk_version": 0, "script": b""}]),
        lambda: (lambda t: at(t, "inputs", len(t["inputs"]) - 1, txid=t["inputs"][0]["txid"], index=t["inputs"][0]["index"]))(_base(rng, n_in=5)),
        lambda: with_(_base(rng), gas=1),
        lambda: with_(_base(rng), subnetwork_id=bytes([2]) + bytes(19)),
        lambda: with_(_base(rng), subnetwork_id=bytes(19) + bytes([1])),
        lambda: with_(_base(rng), version=1),
        lambda: with_(_base(rng), lock_time=T - 1),
        lambda: with_(_base(rng), lock_time=T),
        lambda: with_(_base(rng), lock_time=DAA),
        lambda: with_(_base(rng), lock_time=DAA - 1),
        lambda: with_(_base(rng), lock_time=PMT),
        lambda: with_(_base(rng), lock_time=PMT - 1),
        lambda: (lambda t: with_(t, inputs=[dict(i, sequence=U64) for i in t["inputs"]]))(with_(_base(rng), lock_time=DAA)),
        lambda: (lambda t: with_(t, inputs=[dict(i, sequence=U64) for i in t["inputs"]]))(with_(_base(rng), lock_time=PMT)),
    ]
    return gens


def test_generated_transactions_agree_with_the_oracle(tv):
    """about 10^4 generated transactions, each mutated at one rule's boundary: status, index and both masses equal the oracle's, with the
    test's small limits and again with mass parameters large enough to wrap u64"""
    rng = np.random.default_rng(17)
    gens = _mutants(rng, SMALL)
    txs = [gens[k % len(gens)]() for k in range(10_000)]
    res = _agree(_iso(tv, txs, SMALL), txs, SMALL, "small rules")
    seen = set(int(s) for s in res["status"])
    assert seen >= set(range(14, 32)) - {25} and 0 in seen, sorted(set(range(14, 32)) - seen)  # OutputsValueOverflow cannot be reached
    wrap = dict(SMALL, mass_per_tx_byte=(1 << 63) + 3, mass_per_script_pub_key_byte=U64, mass_per_sig_op=(1 << 62) + 1)
    _agree(_iso(tv, txs[:2000], wrap), txs[:2000], wrap, "wrapping masses")
    _agree(_iso(tv, txs[:2000], SMALL, finality=False), txs[:2000], SMALL, "no finality", finality=False)


def _dup_tx(rng, n, last_pair="dup"):
    t = _base(rng, n_in=n)
    a, b = t["inputs"][-2], t["inputs"][-1]
    if last_pair == "dup":
        b.update(txid=a["txid"], index=a["index"])
    elif last_pair == "txid":
        b.update(txid=a["txid"][:31] + bytes([a["txid"][31] ^ 1]), index=a["index"])
    elif last_pair == "index":
        b.update(txid=a["txid"], index=a["index"] ^ (1 << 31))
    return t


def test_duplicate_inputs(tv):
    """2, 32, 33, 1 000 (and, above the sort's 2 048, 3 000) inputs with the duplicate as the last pair; near-duplicates differing only in the
    last txid byte or the top index byte are not flagged; several large transactions in one launch"""
    rng = np.random.default_rng(3)
    rules = dict(oi.mainnet_rules(), max_tx_inputs=5000)
    txs = []
    for n in (2, 31, 32, 33, 64, 1000, 2048, 2049, 3000):
        for kind in ("dup", "txid", "index", "none"):
            txs.append(_dup_tx(rng, n, kind))
    for t in txs:
        t["lock_time"] = 0
    res = _agree(_iso(tv, txs, rules), txs, rules, "duplicates")
    assert list(res["status"]) == [27, 0, 0, 0] * 9
    # the first and the last input equal, inside a large transaction; and a first-pair duplicate
    t = _base(rng, n_in=1000)
    t["inputs"][-1].update(txid=t["inputs"][0]["txid"], index=t["inputs"][0]["index"])
    u = _base(rng, n_in=700)
    u["inputs"][1].update(txid=u["inputs"][0]["txid"], index=u["inputs"][0]["index"])
    _agree(_iso(tv, [t, u] + txs, rules), [t, u] + txs, rules, "far pairs")


class Mixed:
    """test_gpu_mempool's pool (chains, invalid signatures) plus isolation failures, non-final transactions and feerate thresholds"""

    def __init__(self, pool):
        self.pool = pool
        self.rules = oi.mainnet_rules()
        rng = np.random.default_rng(29)
        base = list(pool.pool)
        txs = []
        for k, t in enumerate(base):
            m = k % 8
            if m == 1:
                t = dict(t, gas=1)
            elif m == 2:
                t = dict(t, inputs=t["inputs"] + [dict(t["inputs"][0])])  # duplicate input
            elif m == 3:
                t = dict(t, lock_time=pool.pov, inputs=[dict(i, sequence=0) for i in t["inputs"]])  # not final at the virtual DAA score
            elif m == 4:
                t = dict(t, lock_time=PMT + 5, inputs=[dict(i, sequence=U64) for i in t["inputs"]])  # final through its sequences
            txs.append(t)
        self.txs = txs
        self.sup = pool.supplied(txs)
        self.thr = np.where(rng.random(len(txs)) < 0.25, 1.0, np.nan)

    def expect(self):
        p = self.pool
        n = len(self.txs)
        iso = [oi.ok_tx_validate(t, self.rules, p.pov, PMT) for t in self.txs]
        ms = np.array([oi.ok_tx_non_contextual_masses(t, self.rules) for t in self.txs], dtype=np.uint64).reshape(-1, 2)
        ok = [ti for ti in range(n) if iso[ti][0] == 0]
        nc = ms.max(axis=1)
        r_ok, m_ok, f_ok = oracle_mempool(p.ora, p.ost, [self.txs[i] for i in ok], [self.sup[i] for i in ok], p.pov, p.op, self.thr[ok], nc[ok])
        res = np.zeros(n, dtype=RESULT_DTYPE)
        mass = np.zeros(n, dtype=np.uint64)
        finals = []
        per_ok = {}
        k = 0
        for j, ti in enumerate(ok):
            res[ti], mass[ti] = r_ok[j], m_ok[j]
            per_ok[ti] = f_ok[k:k + len(self.txs[ti]["inputs"])]
            k += len(self.txs[ti]["inputs"])
        for ti in range(n):
            if iso[ti][0]:
                res[ti]["status"], res[ti]["fail_input"] = iso[ti]
                finals.extend(self.sup[ti])
            else:
                finals.extend(per_ok[ti])
        return (res, mass, finals), ok, iso, ms, nc

    def run(self, tv):
        b, mask = _batch(self.txs, self.sup)
        return tv.validate_mempool_transactions_in_parallel_full(self.pool.us, b, self.pool.pov, PMT, TxRules(), self.thr, supplied=mask)


@pytest.fixture
def pool(gpu_ctx, oracle):
    p = Pool(gpu_ctx, oracle)
    yield p
    p.close()


def test_mempool_full_pipeline(pool):
    """isolation -> finality -> the UTXO-context pipeline equals the oracle; on the transactions that pass the first two stages the new call
    and kgv_validate_mempool_txs (fed the oracle's masses) give identical bytes; rejected transactions keep the caller's entries or absent rows"""
    mx = Mixed(pool)
    got = mx.run(pool.tv)
    (er, em, ef), ok, iso, ms, nc = mx.expect()
    res, mass, masses, ent, arena = got
    same((res, mass, ent, arena), (er, em, ef), "full")
    assert (masses["compute_mass"] == ms[:, 0]).all() and (masses["transient_mass"] == ms[:, 1]).all()
    st = set(int(s) for s in res["status"])
    assert {0, 1, 13, 27, 28, 31} <= st and (9 in st or 10 in st), st
    rejected = [ti for ti in range(len(mx.txs)) if iso[ti][0]]
    assert (mass[rejected] == 0).all() and (res["fee"][rejected] == 0).all()
    assert [int(res["fail_input"][ti]) for ti in rejected] == [iso[ti][1] for ti in rejected]
    # the same transactions through the pre-existing call, with the oracle's masses as the caller's non-contextual mass
    sub = [mx.txs[i] for i in ok]
    old = pool.tv.validate_mempool_transactions_in_utxo_context(pool.us, _batch(sub, [mx.sup[i] for i in ok])[0], pool.pov, mx.thr[ok], nc[ok],
                                                                supplied=_batch(sub, [mx.sup[i] for i in ok])[1])
    assert res[ok].tobytes() == old[0].tobytes() and mass[ok].tobytes() == old[1].tobytes()
    # rejected transactions' rows: the caller's entry, or absent - never a looked-up one
    k = 0
    for ti, t in enumerate(mx.txs):
        rows = ent[k:k + len(t["inputs"])]
        k += len(t["inputs"])
        if not iso[ti][0]:
            continue
        for e, s in zip(rows, mx.sup[ti]):
            if s is None:
                assert e["pad_"][0] == 1 and e["amount"] == 0, ti
            else:
                assert e["pad_"][0] == 0 and int(e["amount"]) == s["amount"], ti
    # an in-set outpoint of a rejected transaction would have been found: it is absent here
    looked = [ti for ti in rejected if any(s is None and pool.ost.get(_key36(i)) is not None for i, s in zip(mx.txs[ti]["inputs"], mx.sup[ti]))]
    assert looked


def test_rejected_transactions_never_reach_the_sigcache(pool):
    """with a SigCache attached, the full call makes exactly the lookups and inserts the pre-existing call makes on the transactions that pass
    isolation and finality"""
    mx = Mixed(pool)
    (er, _, _), ok, iso, ms, nc = mx.expect()
    ctx = pool.tv.ctx
    sc = SigCache(ctx, 1 << 16)
    sc.attach()
    try:
        mx.run(pool.tv)
        c_full = sc.counters()
        sc.clear()
        c0 = sc.counters()
        sub = [mx.txs[i] for i in ok]
        b, mask = _batch(sub, [mx.sup[i] for i in ok])
        pool.tv.validate_mempool_transactions_in_utxo_context(pool.us, b, pool.pov, mx.thr[ok], nc[ok], supplied=mask)
        c_sub = sc.counters()
        assert c_full["lookups"] == c_sub["lookups"] - c0["lookups"] > 0, (c_full, c_sub, c0)
        assert c_full["inserts"] == c_sub["inserts"] - c0["inserts"] > 0, (c_full, c_sub, c0)
    finally:
        sc.close()


def test_nonstandard_scripts_after_isolation(gpu_ctx, oracle):
    """spends the fast path declines (decided by the device script engine) pass isolation and are decided as by kgv_validate_mempool_txs"""
    from rusty_kaspa_b200 import GpuUtxoSet, Params, TransactionValidator
    from test_gpu_host_vm import _custom_spends
    txs, ents = _custom_spends(48, seed=5)
    us = GpuUtxoSet(gpu_ctx, 1 << 10)
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=0, storage_mass_parameter=0))
    b, mask = _batch(txs, ents)
    full = tv.validate_mempool_transactions_in_parallel_full(us, b, 1000, PMT, TxRules(), supplied=mask)
    old = tv.validate_mempool_transactions_in_utxo_context(us, b, 1000, supplied=mask)
    iso = [oi.ok_tx_validate(t, oi.mainnet_rules(), 1000, PMT) for t in txs]
    for ti, (s, _) in enumerate(iso):
        if s:
            assert full[0]["status"][ti] == s
        else:
            assert full[0][ti].tobytes() == old[0][ti].tobytes(), ti
    assert sum(1 for s, _ in iso if s == 0) > 20 and (full[0]["status"] == 0).any()
    us.close()
