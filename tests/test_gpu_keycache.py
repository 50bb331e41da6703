"""The device key cache (kgv_keycache): comb-form key records kept across the verify launches of one context.  Every verdict is compared
with the CPU oracle and with the same call made without the cache, for both kinds, in small launches (at most one item per resident
thread: the misses are stored after the verification) and large ones (stored before it), cold, warm and half stored; the joint
ladder's exceptional cases through stored records in one-item calls (the hits counter counts the items the stored-record launch
verifies); key identity; capacity and eviction; kgv_validate_txs, kgv_validate_mempool_txs, kgv_check_scripts, replay windows with and
without a SigCache, and a sharded replay with a cache per rank; and the API's refusals."""
import numpy as np
import pytest

import joint_model as J
import ladder_model as L
from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

P = 2**256 - 2**32 - 977
LARGE = 60_000  # more items than an H100's 50 688 resident verify threads


@pytest.fixture
def ctx():
    import rusty_kaspa_b200 as rk
    c = rk.GpuContext(0)
    yield c
    c.close()


def _kc(ctx, s=1 << 12, e=1 << 12):
    from rusty_kaspa_b200.validator import KeyCache
    return KeyCache(ctx, s, e)


def _triples(kind, n, seed, n_keys):
    gen = W.ecdsa_triples if kind == "ecdsa" else W.schnorr_triples
    pk, msg, sig, _ = gen(n, seed=seed, n_keys=n_keys, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05)
    if kind == "schnorr" and n >= 16:  # unparseable keys: x >= p and x off the curve
        rng = np.random.default_rng(seed)
        pk[1] = np.frombuffer((P + 5).to_bytes(32, "big"), np.uint8)
        pk[3] = np.frombuffer(W._non_residue_x(rng).to_bytes(32, "big"), np.uint8)
    if kind == "ecdsa" and n >= 16:  # a bad tag and an off-curve x
        pk[1, 0] = 0x05
        pk[3, 1:] = np.frombuffer(W._non_residue_x(np.random.default_rng(seed)).to_bytes(32, "big"), np.uint8)
    return pk, msg, sig


def _verify(ctx, kind, pk, msg, sig):
    return (ctx.verify_ecdsa_batch if kind == "ecdsa" else ctx.verify_schnorr_batch)(pk, msg, sig)


def _oracle(oracle, kind, pk, msg, sig):
    return (oracle_ecdsa_batch if kind == "ecdsa" else oracle_schnorr_batch)(oracle, pk, msg, sig)


def _check(ctx, oracle, kind, pk, msg, sig, plain=None):
    got = _verify(ctx, kind, pk, msg, sig)
    exp = _oracle(oracle, kind, pk, msg, sig)
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at {bad[:5]}: got {got[bad[:5]]} exp {exp[bad[:5]]}"
    if plain is not None:
        assert (got == plain).all()
    return got


def _consistent(kc, ecdsa, capacity):
    c = kc.counters(ecdsa)
    assert c["hits"] <= c["lookups"] and 0 <= c["inserts"] - c["evictions"] <= capacity, c
    return c


@pytest.mark.parametrize("kind", ["schnorr", "ecdsa"])
@pytest.mark.parametrize("n", [1, 16, 256, LARGE])
def test_cold_warm_and_half(ctx, oracle, kind, n):
    import rusty_kaspa_b200 as rk
    n_keys = max(1, n // 8)
    pk, msg, sig = _triples(kind, n, 100 + n, n_keys)
    pk2, msg2, sig2 = _triples(kind, n, 200 + n, n_keys)
    half = n // 2
    mix = [np.concatenate([a[:half], b[half:]]) for a, b in ((pk, pk2), (msg, msg2), (sig, sig2))]
    ref = rk.GpuContext(0)
    try:
        plain = [_verify(ref, kind, *t) for t in ((pk, msg, sig), tuple(mix))]
    finally:
        ref.close()
    cap = 1 << 15  # sets of eight at most a quarter full: every key of a call finds a slot
    kc = _kc(ctx, cap, cap)
    e = kind == "ecdsa"
    try:
        _check(ctx, oracle, kind, pk, msg, sig, plain[0])                    # cold: every key a miss
        c0 = _consistent(kc, e, cap)
        assert c0["lookups"] == n and c0["inserts"] >= 1
        if n == LARGE:  # a large launch stores its keys first, then verifies from the stored records
            assert c0["hits"] >= n - n // 1000, c0
        else:  # a small one verifies its misses inline and stores them afterwards
            assert c0["hits"] == 0, c0
        _check(ctx, oracle, kind, pk, msg, sig, plain[0])                    # warm: every key stored
        c1 = _consistent(kc, e, cap)
        # (a key whose eight-way set is full is not stored: at this load a few of 60 000 items at most)
        assert c1["lookups"] == 2 * n and c1["hits"] - c0["hits"] >= n - n // 1000
        _check(ctx, oracle, kind, *mix, plain[1])                            # half stored keys, half new ones
        _consistent(kc, e, cap)
        _check(ctx, oracle, kind, *mix, plain[1])
    finally:
        kc.close()


@pytest.mark.parametrize("kind", ["schnorr", "ecdsa"])
def test_small_calls_reach_the_joint_ladder_edges(ctx, oracle, kind):
    cs = J.ecdsa_joint_cases(oracle) if kind == "ecdsa" else J.schnorr_infinity_and_fix_cases(oracle)
    cpk, cmsg, csig = L.arrays(cs)
    cexp = np.array([c["exp"] for c in cs], dtype=np.uint8)
    assert (_oracle(oracle, kind, cpk, cmsg, csig) == cexp).all()
    kc = _kc(ctx)
    e = kind == "ecdsa"
    try:
        for i in range(len(cs)):
            one = (cpk[i:i + 1], cmsg[i:i + 1], csig[i:i + 1])
            assert _verify(ctx, kind, *one)[0] == cexp[i], cs[i]["label"]     # stores the key
            h = kc.counters(e)["hits"]
            assert _verify(ctx, kind, *one)[0] == cexp[i], cs[i]["label"]     # one item, its stored comb record
            assert kc.counters(e)["hits"] == h + 1, cs[i]["label"]
    finally:
        kc.close()


def test_key_identity(ctx, oracle):
    spk, smsg, ssig, _ = W.schnorr_triples(8, seed=5, n_keys=8, n_nonces=8, frac_bitflip=0.0, frac_adversarial=0.0)
    epk, emsg, esig, _ = W.ecdsa_triples(8, seed=5, n_keys=8, n_nonces=8, frac_bitflip=0.0, frac_adversarial=0.0)
    x = epk[:, 1:].copy()
    e02, e03 = epk.copy(), epk.copy()
    e02[:, 0], e03[:, 0] = 2, 3
    kc = _kc(ctx)
    try:
        for _ in range(2):
            _check(ctx, oracle, "schnorr", x, smsg, ssig)   # the ECDSA keys' x as Schnorr keys
            _check(ctx, oracle, "ecdsa", e02, emsg, esig)
            _check(ctx, oracle, "ecdsa", e03, emsg, esig)
            _check(ctx, oracle, "ecdsa", epk, emsg, esig)
        s, e = kc.counters(False), kc.counters(True)
        ux = len(np.unique(x, axis=0))
        assert s["inserts"] == ux and e["inserts"] == 2 * ux, (s, e)  # 02 and 03 of one x are two keys
        # one-bit neighbours of stored keys never share their records
        near = spk.copy()
        near[:, 31] ^= 1
        for _ in range(2):
            _check(ctx, oracle, "schnorr", near, smsg, ssig)
            _check(ctx, oracle, "schnorr", spk, smsg, ssig)
        nearE = epk.copy()
        nearE[:, 32] ^= 1
        for _ in range(2):
            _check(ctx, oracle, "ecdsa", nearE, emsg, esig)
            _check(ctx, oracle, "ecdsa", epk, emsg, esig)
    finally:
        kc.close()


@pytest.mark.parametrize("n", [256, LARGE])
def test_capacity_and_eviction(ctx, oracle, n):
    kc = _kc(ctx, 16, 16)  # two sets of eight per kind
    try:
        for seed in range(4):  # more distinct keys per call than the partition holds, and new keys every call
            pk, msg, sig = _triples("schnorr", n, 300 + seed, 64)
            _check(ctx, oracle, "schnorr", pk, msg, sig)
            _check(ctx, oracle, "schnorr", pk, msg, sig)
            _consistent(kc, False, 16)
        # a call whose every key hits, then one whose misses would evict them: both correct
        pk, msg, sig = _triples("schnorr", 16, 400, 4)
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        h = kc.counters(False)["hits"]
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        assert kc.counters(False)["hits"] == h + 16
        pk2, msg2, sig2 = _triples("schnorr", 64, 401, 64)
        _check(ctx, oracle, "schnorr", pk2, msg2, sig2)
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        c = _consistent(kc, False, 16)
        assert c["evictions"] > 0
    finally:
        kc.close()


def test_api(ctx, oracle):
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200.validator import KeyCache
    with pytest.raises(rk.KgvError):
        KeyCache(ctx, 0, 0)
    with pytest.raises(rk.KgvError):
        KeyCache(ctx, (1 << 20) + 1, 0)
    with pytest.raises(rk.KgvError):
        ctx._check(ctx._lib.kgv_keycache_clear(ctx._h))  # no cache yet
    kc = KeyCache(ctx, 64, 0)  # no ECDSA partition: ECDSA launches run as without a cache
    try:
        with pytest.raises(rk.KgvError):
            KeyCache(ctx, 64, 0)  # one per context
        pk, msg, sig = _triples("schnorr", 16, 500, 4)
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        epk, emsg, esig = _triples("ecdsa", 16, 500, 4)
        _check(ctx, oracle, "ecdsa", epk, emsg, esig)
        assert kc.counters(True) == dict(lookups=0, hits=0, inserts=0, evictions=0)
        kc.detach()  # off: no lookups, the records stay
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        assert kc.counters(False)["lookups"] == 16
        kc.attach()
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        assert kc.counters(False)["hits"] == 16
        kc.clear()
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        c = kc.counters(False)
        assert c["lookups"] == 16 and c["hits"] == 0, c  # after a clear, only misses
        # a verify launch on a caller's stream: the counters wait for it through the cache's own events
        import torch
        s = torch.cuda.Stream()
        ctx.use_stream(s.cuda_stream)
        _check(ctx, oracle, "schnorr", pk, msg, sig)
        ctx.reset_stream()
        assert kc.counters(False)["hits"] == 16
    finally:
        kc.close()  # destroyed: the context runs on without it
    _check(ctx, oracle, "schnorr", pk, msg, sig)
    assert ctx._lib.kgv_keycache_counter(ctx._h, 0, 0) == 0
    KeyCache(ctx, 64, 64)  # left to kgv_destroy


def _funded(n):
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.txbatch import build_batch
    fk, fe, txs = simgen.funded_window(n, n_keys=32, n_nonces=64, mix=(0.4, 0.2, 0.2, 0.2))
    ents, k = [], 0
    for t in txs:
        ents.append(fe[k:k + len(t["inputs"])])
        k += len(t["inputs"])
    return fk, fe, txs, build_batch(txs), build_batch(txs, ents)


def _window(kc_on, sigcache=False):
    """a funded window with ECDSA and multisig through kgv_validate_txs and kgv_validate_mempool_txs against a UTXO set, and a replay
    window with invalid transactions, each twice"""
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200 import GpuUtxoSet, simgen
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_BLOCK_DTYPE
    from rusty_kaspa_b200.validator import Params, SigCache, TransactionValidator
    ctx = rk.GpuContext(0)
    kc = _kc(ctx) if kc_on else None
    sc = None
    if sigcache:
        sc = SigCache(ctx, 1 << 14)
        sc.attach()
    try:
        out = []
        fk, fe, txs, b, pb = _funded(300)
        us = GpuUtxoSet(ctx, 1 << 12)
        ae, ab = simgen.entries_to_arrays(fe)
        us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
        val = TransactionValidator(ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
        for _ in range(2):
            res = val.validate_transactions_in_parallel(us, b, 10)
            out.append((res["status"].copy(), res["fee"].copy()))
            m = val.validate_mempool_transactions_in_utxo_context(us, b, 10)[0]
            out.append((m["status"].copy(), m["fee"].copy()))
        us.close()
        g = simgen.FastDag(seed=9, n_keys=64, n_nonces=128, coinbase_maturity=3, mix=(0.4, 0.2, 0.2, 0.2), frac_invalid=0.1, coinbase_outputs=8)
        g.generate(24, 12)
        rb, first, pov = g.take()
        arr = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
        arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1
        for _ in range(2):  # the same window twice from an empty UTXO set: the second finds its keys stored
            rp = DagReplayer(ctx, Params(coinbase_maturity=3, storage_mass_parameter=g.C), 1 << 13)
            got, acc = rp.replay_window(rb, arr, want_accept=True)
            out.append((got["status"].copy(), got["script_err"].copy(), acc.copy(), rp.us.digest()))
            rp.close()
        g.close()
        stats = (kc.counters(False), kc.counters(True)) if kc else None
        return out, stats, pb
    finally:
        if sc:
            sc.close()
        if kc:
            kc.close()
        ctx.close()


@pytest.mark.parametrize("sigcache", [False, True])
def test_validation_mempool_and_replay_unchanged(oracle, sigcache):
    import oracle_tx
    from rusty_kaspa_b200 import simgen
    off, _, pb = _window(False, sigcache)
    on, stats, _ = _window(True, sigcache)
    assert len(off) == len(on)
    for a, b in zip(off, on):
        for x, y in zip(a, b):
            assert (np.asarray(x) == np.asarray(y)).all() if not isinstance(x, bytes) else x == y
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    exp = [oracle_tx.validate_populated(oracle, pb, i, 10, 0, op) for i in range(len(pb.txs))]
    for st, fee in (on[0], on[2]):  # kgv_validate_txs, cold and warm
        assert [int(x) for x in st] == [int(e["status"]) for e in exp] and [int(x) for x in fee] == [int(e["fee"]) for e in exp]
    if sigcache:  # the repeated calls are answered by the SigCache: only the first ones reach a verify launch
        assert stats[0]["lookups"] > 0 and stats[0]["inserts"] > 0, stats
    else:
        assert stats[0]["hits"] > 0 and stats[1]["hits"] > 0, stats


def test_check_scripts_on_engine_only_spends(ctx, oracle):
    """kgv_check_scripts (the device script engine's rounds through kgv_verify_items): P2SH envelopes, IF/ELSE and the other custom
    shapes, cold then warm, against the host engine's verdicts"""
    from rusty_kaspa_b200 import Params, TransactionValidator
    from test_gpu_script_engine import _expected, _got, _mixed_window
    txs, ents = _mixed_window(11)
    pb, exp = _expected(oracle, txs, ents)
    tv = TransactionValidator(ctx, Params(coinbase_maturity=0, storage_mass_parameter=0))
    kc = _kc(ctx)
    try:
        for _ in range(2):
            res = tv.validate_populated_transactions(pb, 1000, flags=2)
            assert int((res["status"] == 11).sum()) > 50  # declined by the fast path: the engine decides them
            tv.check_scripts(pb, res)
            assert _got(res) == exp
        c = kc.counters(False)
        assert c["hits"] > 0 and c["inserts"] > 0, c
    finally:
        kc.close()


def test_sharded_replay_with_a_cache_per_rank(oracle):
    """two ranks (one context per GPU, one host thread each) replay the same windows with sharding on, each with its own key cache:
    verdicts, accept masks and replicas equal the oracle's"""
    import threading
    import torch
    if torch.cuda.device_count() < 2:
        # two ranks as contexts of one H100 stop in the peer exchange with or without a key cache (as
        # test_gpu_comm.py::test_sharded_replay_equals_unsharded does there): this needs a GPU per rank
        pytest.skip("needs two GPUs")
    import oracle_tx
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.comm import ShardComm
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_BLOCK_DTYPE
    from rusty_kaspa_b200.validator import KeyCache, Params
    n_ranks = 2
    g = simgen.FastDag(seed=21, n_keys=64, n_nonces=256, coinbase_maturity=3, mix=(0.4, 0.2, 0.2, 0.2), frac_invalid=0.1, coinbase_outputs=12)
    wins = []
    for _ in range(3):
        g.generate(40, 40)
        wins.append(g.take())
    prm = Params(coinbase_maturity=3, storage_mass_parameter=g.C)
    ost = oracle_tx.State(oracle)
    op = oracle_tx.params(coinbase_maturity=3, storage_mass_parameter=g.C)
    exp = [oracle_tx.state_replay(ost, b, first, pov, op, threads=8) for b, first, pov in wins]

    def blocks(first, pov):
        arr = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
        arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1
        return arr
    ctxs = [rk.GpuContext(r % torch.cuda.device_count()) for r in range(n_ranks)]
    kcs = [KeyCache(c, 1 << 12, 1 << 12) for c in ctxs]
    comms = [ShardComm(ctxs[r], n_ranks, r, slice_capacity=1 << 20) for r in range(n_ranks)]
    ShardComm.connect_local(comms)
    reps = [DagReplayer(ctxs[r], prm, 1 << 16) for r in range(n_ranks)]
    res, errs = [None] * n_ranks, []

    def body(r):
        try:
            comms[r].shard_validation(True)
            out = [reps[r].replay_window(b, blocks(first, pov), want_accept=True) for b, first, pov in wins]
            res[r] = (out, reps[r].us.count(), reps[r].us.digest(), kcs[r].counters(False))
        except Exception as e:  # noqa: BLE001
            errs.append((r, e))
    th = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(n_ranks)]
    [t.start() for t in th]
    [t.join(timeout=120) for t in th]
    assert not errs, errs
    assert not any(t.is_alive() for t in th), "a rank did not finish"
    for r in range(n_ranks):
        out, cnt, dig, ctr = res[r]
        for (got, acc), (e, eacc) in zip(out, exp):
            assert (got["status"] == e["status"]).all() and (got["script_err"] == e["script_err"]).all() and (acc == eacc).all()
        assert cnt == ost.count() and dig == ost.digest()
        assert ctr["lookups"] > 0 and ctr["hits"] > 0, ctr
    assert res[0][2] == res[1][2]
    for c in comms:
        c.close()
    for rp in reps:
        rp.close()
    for kc in kcs:
        kc.close()
    for c in ctxs:
        c.close()
    ost.close(); g.close()
