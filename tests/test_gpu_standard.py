"""The mempool's standardness policy on the GPU (kgv_check_txs_standard_in_isolation, kgv_check_txs_standard_in_context, kgv_outputs_dust,
kgv_validate_mempool_txs_with_policy) against the CPU restatement (oracle_standard.py) and the reference's own cases.

The fused call's expectation is composed in the mempool's admission order (validate_and_insert_transaction.rs:20-33, 142-159): the oracle's
standardness in isolation on the oracle's non-contextual masses, then test_gpu_isolation's composed consensus expectation, then the oracle's
standardness in context for the transactions still Ok, on their final entries, storage masses and fees."""
import ctypes

import numpy as np
import pytest

import oracle_isolation as oi
import oracle_standard as os_
from rusty_kaspa_b200 import KgvError, MempoolPolicy, TransactionValidator
from rusty_kaspa_b200.txbatch import build_batch
from rusty_kaspa_b200.validator import RESULT_DTYPE, TX_MASSES_DTYPE, SigCache, TxRules
from test_gpu_isolation import PMT, Mixed
from test_gpu_mempool import Pool

pytestmark = pytest.mark.gpu

U64 = 2**64 - 1
P2PK = bytes([0x20]) + bytes([1] * 32) + bytes([0xac])
P2PK_ECDSA = bytes([0x21]) + bytes([2] * 33) + bytes([0xab])
P2SH = bytes([0xaa, 0x20]) + bytes([3] * 32) + bytes([0x87])
INDEXED = (35, 36, 37, 38, 40, 41)


@pytest.fixture
def tv(gpu_ctx):
    return TransactionValidator(gpu_ctx)


def _policy(p):
    return MempoolPolicy(p.fee, p.min_version, p.max_version)


def _masses(ms):
    m = np.zeros(len(ms), dtype=TX_MASSES_DTYPE)
    m["compute_mass"], m["transient_mass"] = [x[0] for x in ms], [x[1] for x in ms]
    return m


def _device(gpu_ctx, call, b, host_arrays, out_sizes, with_entries=False):
    """one of the standalone calls with the batch, the inputs and the outputs in device memory"""
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    t = {k: dev(v) for k, v in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", b.entries), ("arena", b.arena))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(b.txs), t["inputs"].data_ptr(), len(b.inputs), t["outputs"].data_ptr(), len(b.outputs),
                     t["entries"].data_ptr() if with_entries else None, t["arena"].data_ptr(), len(b.arena))
    ins = [dev(a) for a in host_arrays]
    outs = [torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda") for n in out_sizes]
    rc = call(ctypes.byref(cb), [x.data_ptr() for x in ins], [x.data_ptr() for x in outs])
    gpu_ctx._check(rc)
    gpu_ctx._check(gpu_ctx._lib.kgv_synchronize(gpu_ctx._h))
    return [x.cpu().numpy() for x in outs]


def iso_both(tv, gpu_ctx, txs, ms, pol):
    """host and device pointers give the same bytes; returns the host result"""
    b = build_batch(txs)
    m = _masses(ms)
    res, det = tv.check_transaction_standard_in_isolation(b, m, pol)
    L = gpu_ctx._lib
    dres, ddet = _device(gpu_ctx, lambda cb, i, o: L.kgv_check_txs_standard_in_isolation(gpu_ctx._h, cb, ctypes.byref(pol), i[0], o[0], o[1]), b, [m],
                         [16 * len(txs), 8 * len(txs)])
    assert dres[:16 * len(txs)].tobytes() == res.tobytes() and ddet[:8 * len(txs)].tobytes() == det.tobytes()
    return res, det


def ctx_both(tv, gpu_ctx, txs, entries, ms, smass, fee, pol):
    b = build_batch(txs, entries)
    m, sm, fe = _masses(ms), np.array(smass, dtype=np.uint64), np.array(fee, dtype=np.uint64)
    res, det = tv.check_transaction_standard_in_context(b, m, sm, fe, pol)
    L = gpu_ctx._lib
    dres, ddet = _device(gpu_ctx, lambda cb, i, o: L.kgv_check_txs_standard_in_context(gpu_ctx._h, cb, ctypes.byref(pol), i[0], i[1], i[2], o[0], o[1]), b,
                         [m, sm, fe], [16 * len(txs), 8 * len(txs)], with_entries=True)
    assert dres[:16 * len(txs)].tobytes() == res.tobytes() and ddet[:8 * len(txs)].tobytes() == det.tobytes()
    return res, det


def agree_iso(res, det, txs, ms, p, what=""):
    for k, (t, m) in enumerate(zip(txs, ms)):
        e = os_.check_in_isolation(t, m[0], m[1], p)
        assert (int(res["status"][k]), int(res["fail_input"][k]), int(det[k])) == e, (what, k, e)
    assert (res["fee"] == 0).all() and (res["script_err"] == 0).all()


def agree_ctx(res, det, txs, entries, ms, smass, fee, p, what=""):
    for k, t in enumerate(txs):
        e = os_.check_in_context(t, entries[k], smass[k], ms[k][0], fee[k], p)
        assert (int(res["status"][k]), int(res["fail_input"][k]), int(det[k])) == e, (what, k, e)
    assert [int(x) for x in res["fee"]] == [int(x) for x in fee]


def _tx(n_in=1, n_out=1, sig=b"\x00" * 65, value=10**8, script=P2PK, version=0):
    return {"version": version, "lock_time": 0, "subnetwork_id": bytes(20), "gas": 0, "payload": b"", "mass": 0,
            "inputs": [{"txid": bytes([k % 256]) * 32, "index": k, "sigscript": sig, "sequence": U64, "sig_op_count": 1} for k in range(n_in)],
            "outputs": [{"value": value, "spk_version": 0, "script": script} for _ in range(n_out)]}


def _ent(script=P2PK, version=0):
    return {"amount": 10**9, "spk_version": version, "script": script, "block_daa_score": 0, "is_coinbase": False}


# ---- 1. the reference's cases
def test_reference_cases(tv, gpu_ctx):
    g = os_.golden()
    cases = g["isolation"]["cases"]
    txs = [os_.tx_from_golden(c["tx"]) for c in cases]
    ms = [(c["compute_mass"], c["transient_mass"]) for c in cases]
    res, det = iso_both(tv, gpu_ctx, txs, ms, MempoolPolicy())
    agree_iso(res, det, txs, ms, os_.Policy(), "golden isolation")
    assert [os_.NAME[int(s)] for s in res["status"]] == [os_.ISOLATION_EXPECTED[c["name"]][0] for c in cases]
    # dust rows: one call per relay fee, host and device
    for r in g["dust"]["rows"]:
        b = build_batch([_tx(value=r["value"], script=bytes.fromhex(r["script"]))])
        got = tv.is_transaction_output_dust(b, r["minimum_relay_transaction_fee"])
        L = gpu_ctx._lib
        d = _device(gpu_ctx, lambda cb, i, o: L.kgv_outputs_dust(gpu_ctx._h, cb, r["minimum_relay_transaction_fee"], o[0]), b, [], [1])
        assert bool(got[0]) == r["is_dust"] == bool(d[0]), r["name"]
    # relay-fee rows: one standard input, compute mass = size, the fee one below the minimum and at it
    for r in g["relay_fee"]["rows"]:
        p = os_.Policy(minimum_relay_transaction_fee=r["minimum_relay_transaction_fee"])
        txs = [_tx(), _tx()]
        fee = [r["want"] - 1, r["want"]]
        res, det = ctx_both(tv, gpu_ctx, txs, [[_ent()], [_ent()]], [(r["size"], 0)] * 2, [0, 0], fee, _policy(p))
        assert [int(s) for s in res["status"]] == [42, 0] and [int(x) for x in det] == [r["want"], 0], r["name"]


# ---- 2. the boundaries of every rule
def test_isolation_boundaries(tv, gpu_ctx):
    p = os_.Policy(minimum_relay_transaction_fee=1000, minimum_standard_transaction_version=2, maximum_standard_transaction_version=5)
    M = os_.MAXIMUM_STANDARD_TRANSACTION_MASS
    rows = [(_tx(version=v), (1000, 1000)) for v in (1, 2, 5, 6)]
    rows += [(_tx(version=2), m) for m in ((M, M), (M + 1, 0), (0, M + 1), (M + 1, M + 1))]
    rows += [(_tx(version=3, sig=bytes(n)), (1, 1)) for n in (1650, 1651)]
    t = _tx(version=3, n_out=3)
    t["outputs"][2]["spk_version"] = 1
    rows.append((t, (1, 1)))
    t = _tx(version=3, n_out=3)
    t["outputs"][1]["script"] = P2PK[:-1] + b"\xab"
    t["outputs"][2]["spk_version"] = 1
    rows.append((t, (1, 1)))
    edge = -(-1000 * 3 * (8 + 2 + 8 + 34 + 148) // 1000)
    rows += [(_tx(version=3, value=v), (1, 1)) for v in (edge - 1, edge, 0, U64)]
    rows += [(_tx(version=3, script=s, value=10**8), (1, 1)) for s in (P2PK_ECDSA, P2SH, b"\x6a" + P2PK[1:], P2PK[:1] + b"\x6a" + P2PK[2:])]
    # 1 000 inputs and 1 000 outputs, the offender in the last chunk
    big = _tx(version=3, n_in=1000, n_out=1000)
    big["inputs"][999]["sigscript"] = bytes(1651)
    rows.append((big, (1, 1)))
    big = _tx(version=3, n_in=1000, n_out=1000)
    big["outputs"][990]["value"] = 1
    rows.append((big, (1, 1)))
    txs, ms = [r[0] for r in rows], [r[1] for r in rows]
    res, det = iso_both(tv, gpu_ctx, txs, ms, _policy(p))
    agree_iso(res, det, txs, ms, p, "boundaries")
    assert set(int(s) for s in res["status"]) == {0} | set(range(32, 39))
    assert (int(res["status"][-2]), int(res["fail_input"][-2])) == (35, 999) and (int(res["status"][-1]), int(res["fail_input"][-1])) == (38, 990)


def test_context_boundaries_and_quirk_order(tv, gpu_ctx):
    p = os_.Policy()
    push = lambda d: (bytes([len(d)]) if len(d) <= 75 else bytes([0x4c, len(d)])) + d
    ns = _ent(b"\x51")
    rows = [  # (tx, entries, (compute, transient), storage, fee)
        (_tx(n_in=2), [ns, _ent()], (1000, 0), 0, 0),           # input 0 non-standard, low fee: the input
        (_tx(n_in=2), [_ent(), ns], (1000, 0), 0, 0),           # input 1 non-standard, low fee: the fee
        (_tx(n_in=2), [_ent(), ns], (1000, 0), 0, 1000),        # fee met: input 1
        (_tx(n_in=0), [], (1000, 0), 0, 0),                      # no inputs: no fee check
        (_tx(), [_ent()], (1000, 0), 100_000, 1000),
        (_tx(), [_ent()], (1000, 0), 100_001, 1000),
        (_tx(), [_ent(version=1)], (1000, 0), 0, 1000),
        (_tx(), [_ent(P2PK_ECDSA)], (1000, 0), 0, 1000),
        (_tx(), [_ent()], (999, 0), 0, 998),                      # mass * fee / 1000 = 999
        (_tx(), [_ent()], (0, 0), 0, 999),                        # floor: 0 -> the relay fee itself
        (_tx(), [_ent()], (100_000, 0), 0, U64),
    ]
    for n_ops in (15, 16):
        rows.append((_tx(sig=push(b"\xac" * n_ops)), [_ent(P2SH)], (1000, 0), 0, 1000))
    rows.append((_tx(sig=push(b"\x60\xae")), [_ent(P2SH)], (1000, 0), 0, 1000))
    rows.append((_tx(sig=b"\x61" + push(b"\xac" * 16)), [_ent(P2SH)], (1000, 0), 0, 1000))
    big = _tx(n_in=1000)
    rows.append((big, [_ent()] * 999 + [ns], (1000, 0), 0, 1000))
    txs, ents = [r[0] for r in rows], [r[1] for r in rows]
    ms, sm, fee = [r[2] for r in rows], [r[3] for r in rows], [r[4] for r in rows]
    res, det = ctx_both(tv, gpu_ctx, txs, ents, ms, sm, fee, MempoolPolicy())
    agree_ctx(res, det, txs, ents, ms, sm, fee, p, "context")
    assert [int(s) for s in res["status"][:4]] == [40, 42, 40, 0] and int(res["fail_input"][2]) == 1
    assert (int(res["status"][-1]), int(res["fail_input"][-1])) == (40, 999)
    # the MAX_SOMPI cap, and the overflow of mass * fee
    # (mass * fee fits u64, so mass * fee / 1000 never passes MAX_SOMPI: only the floor's fee itself can be capped)
    cap = MempoolPolicy(minimum_relay_transaction_fee=U64)
    r, d = ctx_both(tv, gpu_ctx, [_tx(), _tx()], [[_ent()], [_ent()]], [(0, 0), (0, 0)], [0, 0], [os_.MAX_SOMPI - 1, os_.MAX_SOMPI], cap)
    assert [int(s) for s in r["status"]] == [42, 0] and int(d[0]) == os_.MAX_SOMPI
    with pytest.raises(KgvError):
        tv.check_transaction_standard_in_context(build_batch([_tx()], [[_ent()]]), _masses([(2, 0)]), np.zeros(1, np.uint64), np.zeros(1, np.uint64), cap)
    # an overflow in a tx whose fee check is never reached (input 0 non-standard) is no error, as in the reference
    r, _ = ctx_both(tv, gpu_ctx, [_tx()], [[ns]], [(2, 0)], [0], [0], cap)
    assert int(r["status"][0]) == 40


# ---- 3. generated transactions
def _pick(rng, xs):
    return xs[int(rng.integers(0, len(xs)))]


def _random(rng, k):
    n_in, n_out = int(rng.integers(1, 5)), int(rng.integers(1, 5))
    spks = [P2PK, P2PK_ECDSA, P2SH]
    t = _tx(n_in, n_out, version=int(rng.integers(0, 2)) if rng.random() < 0.1 else 0)
    ents = [_ent(spks[int(rng.integers(0, 3))]) for _ in range(n_in)]
    for o in t["outputs"]:
        o["script"] = spks[int(rng.integers(0, 3))]
        o["value"] = _pick(rng, [600, 606, 605, 10**8, U64, 0])
    for _ in range(int(rng.integers(0, 3))):  # one or more mutations
        m = int(rng.integers(0, 8))
        i, o = int(rng.integers(0, n_in)), int(rng.integers(0, n_out))
        if m == 0:
            t["inputs"][i]["sigscript"] = bytes(_pick(rng, [1650, 1651, 3000]))
        elif m == 1:
            t["outputs"][o]["spk_version"] = 1
        elif m == 2:
            t["outputs"][o]["script"] = bytes(rng.bytes(int(rng.integers(0, 40))))
        elif m == 3:
            ents[i] = _ent(bytes(rng.bytes(int(rng.integers(30, 37)))))
        elif m == 4:
            ents[i] = _ent(P2SH)
            t["inputs"][i]["sigscript"] = bytes([0x51]) + bytes([int(rng.integers(1, 40))]) + rng.bytes(int(rng.integers(0, 40)))
        elif m == 5:
            ents[i] = _ent(P2SH)
            body = bytes(_pick(rng, [0xac, 0xae, 0x53, 0x60, 0xab, 0x00]) for _ in range(int(rng.integers(1, 25))))
            t["inputs"][i]["sigscript"] = bytes([len(body)]) + body
        elif m == 6:
            ents[i] = _ent(P2PK, version=1)
        else:
            t["outputs"][o]["script"] = b"\x6a" + t["outputs"][o]["script"][1:]
    ms = (_pick(rng, [1000, 99_999, 100_000, 100_001]), _pick(rng, [1000, 100_000, 100_001]))
    return t, ents, ms, _pick(rng, [0, 1000, 100_000, 100_001]), _pick(rng, [0, 999, 1000, 10**6, 10**9])


def test_generated_transactions_agree_with_the_oracle(tv, gpu_ctx):
    rng = np.random.default_rng(41)
    rows = [_random(rng, k) for k in range(10_000)]
    txs, ents = [r[0] for r in rows], [r[1] for r in rows]
    ms, sm, fee = [r[2] for r in rows], [r[3] for r in rows], [r[4] for r in rows]
    p = os_.Policy(minimum_relay_transaction_fee=1000)
    res, det = tv.check_transaction_standard_in_isolation(build_batch(txs), _masses(ms), _policy(p))
    agree_iso(res, det, txs, ms, p, "generated isolation")
    assert set(int(s) for s in res["status"]) == {0} | set(range(32, 39))
    res, det = tv.check_transaction_standard_in_context(build_batch(txs, ents), _masses(ms), np.array(sm, np.uint64), np.array(fee, np.uint64), _policy(p))
    agree_ctx(res, det, txs, ents, ms, sm, fee, p, "generated context")
    assert set(int(s) for s in res["status"]) == {0, 39, 40, 41, 42}
    # every output of the batch through kgv_outputs_dust (one thread per output, flat indexing, a partial last block)
    outs = [o for t in txs for o in t["outputs"]]
    assert len(outs) % 256 != 0
    for f in (0, 1, 1000, 10**6, U64):
        got = tv.is_transaction_output_dust(build_batch(txs), f)
        exp = np.array([os_.is_transaction_output_dust(o["value"], o["script"], f) for o in outs])
        assert len(got) == len(outs) and (got == exp).all(), (f, np.nonzero(got != exp)[0][:5])


# ---- 4. the fused call
@pytest.fixture
def pool(gpu_ctx, oracle):
    p = Pool(gpu_ctx, oracle)
    yield p
    p.close()


class MixedStd(Mixed):
    """test_gpu_isolation's mixed mempool batch plus transactions that fail standardness in isolation"""

    def __init__(self, pool):
        super().__init__(pool)
        for k, t in enumerate(self.txs):
            if k % 11 == 5:
                self.txs[k] = dict(t, outputs=[dict(o, spk_version=1) for o in t["outputs"]])
            elif k % 11 == 7:
                self.txs[k] = dict(t, inputs=[dict(t["inputs"][0], sigscript=bytes(1651))] + t["inputs"][1:])

    def expect_std(self, policy, ent):
        p = self.pool
        n = len(self.txs)
        ms = [oi.ok_tx_non_contextual_masses(t, self.rules) for t in self.txs]
        st_iso = [os_.check_in_isolation(t, m[0], m[1], policy) for t, m in zip(self.txs, ms)]
        keep = [ti for ti in range(n) if st_iso[ti][0] == 0]
        sub = Mixed.__new__(Mixed)
        sub.pool, sub.rules, sub.txs = p, self.rules, [self.txs[i] for i in keep]
        sub.sup, sub.thr = [self.sup[i] for i in keep], self.thr[keep]
        (r_k, m_k, _), _, _, _, _ = sub.expect()
        res = np.zeros(n, dtype=RESULT_DTYPE)
        mass = np.zeros(n, dtype=np.uint64)
        det = np.zeros(n, dtype=np.uint64)
        for j, ti in enumerate(keep):
            res[ti], mass[ti] = r_k[j], m_k[j]
        for ti in range(n):
            if st_iso[ti][0]:
                res[ti]["status"], res[ti]["fail_input"], det[ti] = st_iso[ti]
        # standardness in context on the final entries the call returned (equal to the oracle's: checked by the caller)
        k = 0
        for ti, t in enumerate(self.txs):
            rows = ent[k:k + len(t["inputs"])]
            k += len(t["inputs"])
            if res[ti]["status"] != 0:
                continue
            ents = [{"spk_version": int(e["spk_version"]), "script": bytes(self.arena[int(e["script_off"]):int(e["script_off"]) + int(e["script_len"])])}
                    for e in rows]
            s = os_.check_in_context(t, ents, int(mass[ti]), ms[ti][0], int(res[ti]["fee"]), policy)
            if s[0]:
                res[ti]["status"], res[ti]["fail_input"], det[ti] = s
        return res, mass, det, keep, st_iso


def test_fused_call_agrees_with_the_composed_oracle(pool, gpu_ctx):
    mx = MixedStd(pool)
    b, mask = __import__("test_gpu_mempool")._batch(mx.txs, mx.sup)
    tv = pool.tv
    launches = lambda: int(gpu_ctx._lib.kgv_launch_count(gpu_ctx._h))
    # policy = None: byte-identical to kgv_validate_mempool_txs_in_parallel, and two launches fewer than with a policy
    c0 = launches()
    base = tv.validate_mempool_transactions_in_parallel_full(pool.us, b, pool.pov, PMT, TxRules(), mx.thr, supplied=mask)
    c1 = launches()
    none = tv.validate_mempool_transactions_with_policy(pool.us, b, pool.pov, PMT, None, TxRules(), mx.thr, supplied=mask)
    c2 = launches()
    for a, z in zip(base, none[:5]):
        assert a.tobytes() == z.tobytes()
    assert (none[5] == 0).all() and c2 - c1 == c1 - c0
    # a relay fee that a part of the accepted transactions falls short of (at least 1 sompi/kg)
    ok = base[0]["status"] == 0
    rate = base[0]["fee"][ok].astype(float) * 1000 / np.maximum(base[2]["compute_mass"][ok], 1).astype(float)
    p = os_.Policy(minimum_relay_transaction_fee=max(1, int(np.percentile(rate, 25))))
    got = tv.validate_mempool_transactions_with_policy(pool.us, b, pool.pov, PMT, _policy(p), TxRules(), mx.thr, supplied=mask)
    res, mass, masses, ent, arena, det = got
    mx.arena = arena
    er, em, ed, keep, st_iso = mx.expect_std(p, ent)
    assert (res["status"] == er["status"]).all(), [(int(i), int(res["status"][i]), int(er["status"][i])) for i in np.nonzero(res["status"] != er["status"])[0][:8]]
    assert (res["fail_input"] == er["fail_input"])[np.isin(res["status"], INDEXED)].all()
    assert (det == ed).all() and (mass == em).all() and (res["script_err"] == er["script_err"]).all()
    feeful = ~np.isin(res["status"], (1, 2, 3, 4, 5, 6, 12))
    assert (res["fee"][feeful] == er["fee"][feeful]).all()
    assert masses.tobytes() == base[2].tobytes()
    st = set(int(s) for s in res["status"])
    assert {35, 36, 42} <= st and (1 in st or 13 in st), st
    # standardness-rejected in isolation: never looked up (rows = the caller's or absent), storage mass 0
    rej = [ti for ti in range(len(mx.txs)) if st_iso[ti][0]]
    assert rej and (mass[rej] == 0).all()
    # with a SigCache: the lookups and inserts of the transactions that pass standardness in isolation, whatever the context stage says
    sc = SigCache(gpu_ctx, 1 << 16)
    sc.attach()
    try:
        tv.validate_mempool_transactions_with_policy(pool.us, b, pool.pov, PMT, _policy(p), TxRules(), mx.thr, supplied=mask)
        c_pol = sc.counters()
        sc.clear()
        c0 = sc.counters()
        sub = [mx.txs[i] for i in keep]
        sb, smask = __import__("test_gpu_mempool")._batch(sub, [mx.sup[i] for i in keep])
        tv.validate_mempool_transactions_in_parallel_full(pool.us, sb, pool.pov, PMT, TxRules(), mx.thr[keep], supplied=smask)
        c_sub = sc.counters()
        assert c_pol["lookups"] == c_sub["lookups"] - c0["lookups"] > 0 and c_pol["inserts"] == c_sub["inserts"] - c0["inserts"] > 0
    finally:
        sc.close()
    # on a batch the policy rejects nothing of before the scripts, the call makes exactly the two launches of the policy more
    plain = Mixed(pool)
    pb, pmask = __import__("test_gpu_mempool")._batch(plain.txs, plain.sup)
    open_policy = MempoolPolicy(minimum_relay_transaction_fee=0, maximum_standard_transaction_version=0xFFFF)
    c0 = launches()
    r0 = tv.validate_mempool_transactions_in_parallel_full(pool.us, pb, pool.pov, PMT, TxRules(), plain.thr, supplied=pmask)
    c1 = launches()
    r1 = tv.validate_mempool_transactions_with_policy(pool.us, pb, pool.pov, PMT, open_policy, TxRules(), plain.thr, supplied=pmask)
    c2 = launches()
    assert not np.isin(r1[0]["status"], range(32, 39)).any()
    assert c2 - c1 == (c1 - c0) + 2
    # device pointers give the bytes of host pointers: with the policy, without it (detail zeroed), and with a relay fee above
    # u64::MAX / 100 000 (the call then waits for the overflow flag)
    for pol in (_policy(p), None, MempoolPolicy(minimum_relay_transaction_fee=U64 // 50_000)):
        host = tv.validate_mempool_transactions_with_policy(pool.us, b, pool.pov, PMT, pol, TxRules(), mx.thr, supplied=mask)
        devr = _device_fused(gpu_ctx, pool.us, b, mask, pool.pov, PMT, pool.params, mx.thr, pol)
        for name, h, d in zip(("results", "storage mass", "masses", "entries", "scripts", "detail"), host, devr):
            assert h.tobytes() == d.tobytes(), name


def _device_fused(gpu_ctx, us, b, mask, pov, pmt, params, thr, policy):
    """kgv_validate_mempool_txs_with_policy with every array in device memory (the detail array pre-filled with garbage)"""
    import torch
    from rusty_kaspa_b200.txbatch import ENTRY_DTYPE
    from rusty_kaspa_b200.validator import MEMPOOL_ARGS_DTYPE
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    ent = b.entries.copy()
    ent["pad_"][:, 0] = np.where(mask, 0, 1)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    args = np.zeros(len(b.txs), dtype=MEMPOOL_ARGS_DTYPE)
    args["feerate_threshold"] = np.nan if thr is None else thr
    t = {k: dev(v) for k, v in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", ent), ("arena", b.arena), ("args", args))}
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(b.txs), t["inputs"].data_ptr(), len(b.inputs), t["outputs"].data_ptr(), len(b.outputs),
                     t["entries"].data_ptr(), t["arena"].data_ptr(), len(b.arena))
    n, ni = len(b.txs), len(b.inputs)
    res, mass, ms = (torch.zeros(n * k, dtype=torch.uint8, device="cuda") for k in (16, 8, 16))
    det = torch.full((n * 8,), 0xA5, dtype=torch.uint8, device="cuda")
    eo = torch.zeros(max(ni, 1) * 32, dtype=torch.uint8, device="cuda")
    cap = len(b.arena) + 128 * ni
    so = torch.zeros(max(cap, 8), dtype=torch.uint8, device="cuda")
    used = ctypes.c_size_t()
    gpu_ctx._check(gpu_ctx._lib.kgv_validate_mempool_txs_with_policy(gpu_ctx._h, us._h, ctypes.byref(cb), pov, pmt, ctypes.byref(params),
                                                                     ctypes.byref(TxRules()), t["args"].data_ptr(), res.data_ptr(), mass.data_ptr(),
                                                                     ms.data_ptr(), eo.data_ptr(), so.data_ptr(), cap, ctypes.byref(used),
                                                                     None if policy is None else ctypes.byref(policy), det.data_ptr()))
    gpu_ctx._check(gpu_ctx._lib.kgv_synchronize(gpu_ctx._h))
    return (res.cpu().numpy().view(RESULT_DTYPE), mass.cpu().numpy().view(np.uint64), ms.cpu().numpy().view(TX_MASSES_DTYPE),
            eo.cpu().numpy().view(ENTRY_DTYPE)[:ni], so.cpu().numpy()[:used.value], det.cpu().numpy().view(np.uint64))


# spends the device script engine accepts without a signature: a P2SH entry whose redeem script leaves true on the stack, a bare OP_TRUE
def _p2sh(redeem):
    import hashlib
    return bytes([0xaa, 0x20]) + hashlib.blake2b(redeem, digest_size=32).digest() + bytes([0x87]), bytes([len(redeem)]) + redeem


def _spend(entry_script, sigscript, amount, value, sig_op_count=0):
    t = _tx(sig=sigscript, value=value)
    t["inputs"][0]["sig_op_count"] = sig_op_count
    return t, [dict(_ent(entry_script), amount=amount)]


def test_fused_context_stage_rules_and_overflow(gpu_ctx):
    """the fused call's standardness-in-context stage on spends that pass every consensus rule: storage mass, input class, the P2SH
    sig-op bound, the fee, Ok; the relay-fee overflow fails the call, with host and with device pointers"""
    from rusty_kaspa_b200 import GpuUtxoSet, Params
    true_spk, true_ss = _p2sh(b"\x51")
    many_spk, many_ss = _p2sh(b"\x00\x63" + b"\xac" * 16 + b"\x68\x51")  # 16 CHECKSIGs in a branch that never runs
    rows = [
        _spend(true_spk, true_ss, 10**9 + 10**6, 10**9),      # Ok
        _spend(true_spk, true_ss, 2 * 10**6, 10**6),           # storage mass about C / 2 10^6: RejectStorageMass
        _spend(b"\x51", b"", 10**9 + 10**6, 10**9),            # a bare OP_TRUE entry: RejectInputScriptClass
        _spend(many_spk, many_ss, 10**9 + 10**6, 10**9),       # RejectSignatureCount(16)
        _spend(true_spk, true_ss, 10**9 + 1, 10**9),           # fee 1: RejectInsufficientFee
    ]
    txs, ents = [r[0] for r in rows], [r[1] for r in rows]
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=0))
    us = GpuUtxoSet(gpu_ctx, 1 << 10)
    try:
        b = build_batch(txs, ents)
        mask = np.ones(len(b.inputs), bool)
        p = os_.Policy()
        res, mass, masses, ent, arena, det = tv.validate_mempool_transactions_with_policy(us, b, 1000, 0, _policy(p), supplied=mask)
        assert [int(s) for s in res["status"]] == [0, 39, 40, 41, 42], res
        assert int(mass[1]) > 100_000 and int(det[1]) == int(mass[1]) and int(det[3]) == 16
        for k, t in enumerate(txs):
            e = os_.check_in_context(t, [_ent(ents[k][0]["script"])], int(mass[k]), int(masses["compute_mass"][k]), int(res["fee"][k]), p)
            assert (int(res["status"][k]), int(res["fail_input"][k]), int(det[k])) == e, k
        assert [int(f) for f in res["fee"]] == [10**6, 10**6, 10**6, 10**6, 1]
        # the same batch with device pointers
        devr = _device_fused(gpu_ctx, us, b, mask, 1000, 0, tv.params, None, _policy(p))
        assert devr[0].tobytes() == res.tobytes() and devr[5].tobytes() == det.tobytes()
        # compute mass above 50 000 (60 sig-ops) times a relay fee of u64::MAX / 50 000 overflows at the fee check; the output is not dust
        big = [_spend(true_spk, true_ss, 3 * 10**14 + 10**6, 3 * 10**14, sig_op_count=60)]
        bb = build_batch([r[0] for r in big], [r[1] for r in big])
        over = MempoolPolicy(minimum_relay_transaction_fee=U64 // 50_000)
        r, _, m, _, _, _ = tv.validate_mempool_transactions_with_policy(us, bb, 1000, 0, MempoolPolicy(), supplied=np.ones(1, bool))
        assert int(r["status"][0]) == 0 and int(m["compute_mass"][0]) * (U64 // 50_000) > U64
        with pytest.raises(KgvError):
            tv.validate_mempool_transactions_with_policy(us, bb, 1000, 0, over, supplied=np.ones(1, bool))
        with pytest.raises(KgvError):
            _device_fused(gpu_ctx, us, bb, np.ones(1, bool), 1000, 0, tv.params, None, over)
    finally:
        us.close()
