"""One device key cache shared by several contexts (kgv_keycache_share, include/kgv.h "Key cache").  Every verdict is compared with the CPU
oracle and with the same call made without a cache: keys stored by one context are hits for another; the chain tip (mempool calls on one
context, block validation on another, one UTXO set and one key cache); contexts on threads whose inserts evict what the others read, with
the joint ladder's edge cases in every batch; a cold 60 000-item launch beside small warm calls; the lifetime and the API; the device
script engine and a replay window beside mempool calls; the C++ mirror is tests/test_gpu_cpp_shared_keycache.py."""
import threading

import numpy as np
import pytest

import joint_model as J
import ladder_model as L
from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

LARGE = 60_000   # more items than an H100's 50 688 resident verify threads
JOIN_S = 300     # a thread that takes longer has hung: the test fails instead of waiting for ever


@pytest.fixture
def ctxs():
    import rusty_kaspa_b200 as rk
    cs = [rk.GpuContext(0) for _ in range(3)]
    yield cs
    for c in cs:
        c.close()


def _kc(ctx, s=1 << 12, e=1 << 12):
    from rusty_kaspa_b200.validator import KeyCache
    return KeyCache(ctx, s, e)


def _verify(ctx, kind, pk, msg, sig):
    return (ctx.verify_ecdsa_batch if kind == "ecdsa" else ctx.verify_schnorr_batch)(pk, msg, sig)


def _oracle(oracle, kind, pk, msg, sig):
    return (oracle_ecdsa_batch if kind == "ecdsa" else oracle_schnorr_batch)(oracle, pk, msg, sig)


def _triples(kind, n, seed, n_keys, bitflip=0.05, adversarial=0.05):
    gen = W.ecdsa_triples if kind == "ecdsa" else W.schnorr_triples
    pk, msg, sig, _ = gen(n, seed=seed, n_keys=n_keys, n_nonces=256, frac_bitflip=bitflip, frac_adversarial=adversarial)
    return pk, msg, sig


def _plain(kind, *t):
    """the verdicts of a context without a key cache"""
    import rusty_kaspa_b200 as rk
    c = rk.GpuContext(0)
    try:
        return _verify(c, kind, *t)
    finally:
        c.close()


def _edges(oracle, kind):
    cs = J.ecdsa_joint_cases(oracle) if kind == "ecdsa" else J.schnorr_infinity_and_fix_cases(oracle)
    pk, msg, sig = L.arrays(cs)
    return pk, msg, sig, np.array([c["exp"] for c in cs], dtype=np.uint8)


def _hits(kc, kind):
    return kc.counters(kind == "ecdsa")["hits"]


@pytest.mark.parametrize("kind", ["schnorr", "ecdsa"])
@pytest.mark.parametrize("n", [1, 16, 256])
def test_cross_context_hits(ctxs, oracle, kind, n):
    """context A verifies under a set of keys; context B's new signatures under those keys are all hits"""
    a, b = ctxs[0], ctxs[1]
    pk, msg, sig = _triples(kind, 4 * n, 600 + n, max(1, n // 8))
    first = (pk[:2 * n], msg[:2 * n], sig[:2 * n])
    met = {bytes(k) for k in first[0]}
    rest = [i for i in range(2 * n, 4 * n) if bytes(pk[i]) in met][:n]
    assert len(rest) == n
    second = (pk[rest], msg[rest], sig[rest])
    kc = _kc(a, 1 << 15, 1 << 15)
    kb = kc.on(b)
    try:
        for c, t in ((a, first), (b, second)):
            h = _hits(kc, kind)
            got = _verify(c, kind, *t)
            assert (got == _oracle(oracle, kind, *t)).all() and (got == _plain(kind, *t)).all()
        assert _hits(kc, kind) - h == n
    finally:
        kb.close()
        kc.close()


def _funded(seed, n):
    from rusty_kaspa_b200 import simgen
    fk, fe, txs = simgen.funded_window(n, seed=seed, n_keys=24, n_nonces=64, mix=(0.4, 0.2, 0.2, 0.2))
    ents, k = [], 0
    for t in txs:
        ents.append(fe[k:k + len(t["inputs"])])
        k += len(t["inputs"])
    return fk, fe, txs, ents


def _chain_tip(shared):
    """mempool calls on context M, then kgv_validate_txs on block context B, against one UTXO set; one key cache shared (or one per
    context); no SigCache.  Returns the verdicts and the block call's hit deltas."""
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200 import GpuUtxoSet, simgen
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import Params, TransactionValidator
    m, blk = rk.GpuContext(0), rk.GpuContext(0)
    kb = _kc(blk) if shared is not None else None
    km = (kb.on(m) if shared else _kc(m)) if shared is not None else None
    try:
        fk1, fe1, txs1, e1 = _funded(71, 120)  # spends the mempool meets first
        fk2, fe2, txs2, e2 = _funded(72, 60)   # spends by keys it never met
        us = GpuUtxoSet(blk, 1 << 12)
        for fk, fe in ((fk1, fe1), (fk2, fe2)):
            ae, ab = simgen.entries_to_arrays(fe)
            us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
        prm = Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
        tm, tb = TransactionValidator(m, prm), TransactionValidator(blk, prm)
        mres = tm.validate_mempool_transactions_in_utxo_context(us.on(m), build_batch(txs1), 10)[0]
        h0 = (kb.counters(False)["hits"], kb.counters(True)["hits"]) if kb else (0, 0)
        res = tb.validate_transactions_in_parallel(us, build_batch(txs1 + txs2), 10)
        h1 = (kb.counters(False)["hits"], kb.counters(True)["hits"]) if kb else (0, 0)
        us.close()
        return mres["status"].copy(), res["status"].copy(), res["fee"].copy(), (h1[0] - h0[0], h1[1] - h0[1]), build_batch(txs1 + txs2, e1 + e2)
    finally:
        for k in (km, kb):
            if k:
                k.close()
        m.close()
        blk.close()


def test_chain_tip_mempool_then_block(oracle):
    import oracle_tx
    from rusty_kaspa_b200 import simgen
    off = _chain_tip(None)
    sep = _chain_tip(False)
    on = _chain_tip(True)
    for arm in (sep, on):
        for x, y in zip(off[:3], arm[:3]):
            assert (x == y).all()
    pb = off[4]
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    exp = [oracle_tx.validate_populated(oracle, pb, i, 10, 0, op) for i in range(len(pb.txs))]
    assert [int(x) for x in on[1]] == [int(e["status"]) for e in exp] and [int(x) for x in on[2]] == [int(e["fee"]) for e in exp]
    assert (on[1] == 0).sum() > 100
    # the block context's own cache is cold; the shared one holds the keys the mempool met
    assert on[3][0] > sep[3][0] and on[3][1] > sep[3][1], (sep[3], on[3])


def test_concurrent_eviction(ctxs, oracle):
    """three contexts on threads share a cache of two sets per kind: every call's keys collide, so each context's inserts evict what the
    others read.  Batches mix valid signatures, one-bit corruptions and the joint ladder's edge cases; verify and validation calls."""
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import Params, TransactionValidator
    iters, cap = 8, 16
    edges = {k: _edges(oracle, k) for k in ("schnorr", "ecdsa")}
    work = []  # per context: [(kind, triples, expected)] and a populated batch with its expected verdicts
    prm = Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    for t in range(len(ctxs)):
        calls = []
        for it in range(iters):
            for kind in ("schnorr", "ecdsa"):
                pk, msg, sig = _triples(kind, 40, 7000 + 100 * t + it, 20, bitflip=0.2, adversarial=0.1)
                epk, emsg, esig, _ = edges[kind]
                j = (it * 3 + t) % len(epk)
                sl = slice(j, j + 3)
                tr = tuple(np.concatenate([x, y[sl]]) for x, y in ((pk, epk), (msg, emsg), (sig, esig)))
                exp = _oracle(oracle, kind, *tr)
                assert (exp[40:] == edges[kind][3][sl]).all()
                calls.append((kind, tr, exp))
        _, _, txs, ents = _funded(800 + t, 40)
        pb = build_batch(txs, ents)
        calls.append(("txs", pb, TransactionValidator(ctxs[0], prm).validate_populated_transactions(pb, 10)))  # cache off yet
        work.append(calls)
    kc = _kc(ctxs[0], cap, cap)
    handles = [kc] + [kc.on(c) for c in ctxs[1:]]
    errs = []

    def body(t):
        try:
            tv = TransactionValidator(ctxs[t], prm)
            for it in range(3):
                for kind, tr, exp in work[t]:
                    if kind == "txs":
                        got = tv.validate_populated_transactions(tr, 10)
                        assert (got == exp).all(), (t, it, "validation")
                    else:
                        got = _verify(ctxs[t], kind, *tr)
                        bad = np.nonzero(got != exp)[0]
                        assert len(bad) == 0, (t, it, kind, bad[:5], got[bad[:5]], exp[bad[:5]])
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=body, args=(t,), daemon=True) for t in range(len(ctxs))]
    [x.start() for x in th]
    [x.join(timeout=JOIN_S) for x in th]
    assert not any(x.is_alive() for x in th), "a thread did not finish"
    assert not errs, errs
    for e in (False, True):
        c = kc.counters(e)
        assert c["evictions"] > 0 and c["hits"] <= c["lookups"] and 0 <= c["inserts"] - c["evictions"] <= cap, c
    # forced: one-item calls of distinct new keys, one after another over the contexts, each store their key and, once the partition
    # is full, evict one
    before = kc.counters(False)
    pk, msg, sig = _triples("schnorr", 48, 9000, 48, bitflip=0.0, adversarial=0.0)
    first = sorted(np.unique(pk, axis=0, return_index=True)[1])
    for j, i in enumerate(first):
        one = (pk[i:i + 1], msg[i:i + 1], sig[i:i + 1])
        assert _verify(ctxs[j % len(ctxs)], "schnorr", *one)[0] == 1
    after = kc.counters(False)
    k, free = len(first), cap - (before["inserts"] - before["evictions"])
    assert after["inserts"] - before["inserts"] == k and after["evictions"] - before["evictions"] >= k - free, (before, after)
    for h in handles:
        h.close()


def test_large_launch_beside_small_calls(ctxs, oracle):
    """a cold 60 000-item launch (stored first, then verified from the records) on A while B makes small warm calls: verdicts right, and
    the large launch's hits those of a serial run"""
    a, b = ctxs[0], ctxs[1]
    big = _triples("schnorr", LARGE, 31, LARGE // 8)
    small = _triples("schnorr", 256, 32, 32)
    exp_big, exp_small = _oracle(oracle, "schnorr", *big), _oracle(oracle, "schnorr", *small)
    parts = [tuple(x[i:i + 16] for x in small) for i in range(0, 256, 16)]
    reps = 6

    def run(concurrent):
        kc = _kc(a, 1 << 16, 1 << 10)
        kb = kc.on(b)
        try:
            assert (_verify(b, "schnorr", *small) == exp_small).all()  # B's keys stored
            h0 = kc.counters(False)["hits"]
            errs = []

            def smalls():
                try:
                    for _ in range(reps):
                        for i, p in enumerate(parts):
                            assert (_verify(b, "schnorr", *p) == exp_small[16 * i:16 * i + 16]).all()
                except Exception as e:  # noqa: BLE001
                    errs.append(e)
            th = threading.Thread(target=smalls, daemon=True)
            if concurrent:
                th.start()
            got = _verify(a, "schnorr", *big)
            h_big = kc.counters(False)["hits"] - h0
            if not concurrent:
                th.start()
            th.join(timeout=JOIN_S)
            assert not th.is_alive() and not errs, errs
            bad = np.nonzero(got != exp_big)[0]
            assert len(bad) == 0, bad[:5]
            return kc.counters(False)["hits"] - h0, h_big
        finally:
            kb.close()
            kc.close()
    serial_total, serial_big = run(False)
    assert serial_big >= LARGE - LARGE // 1000
    total, _ = run(True)
    assert serial_total == serial_big + 256 * reps
    assert total == serial_total  # every small call hit in both runs: the large launch's hits are the serial run's


def test_lifetime_and_api(ctxs, oracle):
    import torch
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200.validator import KeyCache
    a, b, c = ctxs
    pk, msg, sig = _triples("schnorr", 16, 40, 4)
    exp = _oracle(oracle, "schnorr", pk, msg, sig)
    # refusals
    with pytest.raises(rk.KgvError, match="kgv_keycache_share"):
        b._check(b._lib.kgv_keycache_share(b._h, a._h))  # the holder has no cache
    kc = KeyCache(a, 1 << 16, 64)
    with pytest.raises(rk.KgvError, match="kgv_keycache_share"):
        a._check(a._lib.kgv_keycache_share(a._h, a._h))  # one context
    kb = kc.on(b)
    with pytest.raises(rk.KgvError, match="kgv_keycache_share"):
        kc.on(b)  # b has one already
    with pytest.raises(rk.KgvError):
        KeyCache(b, 64, 64)
    # per-context switch: b off leaves a's lookups on
    kb.detach()
    l0 = kc.counters(False)["lookups"]
    assert (_verify(b, "schnorr", pk, msg, sig) == exp).all()
    assert kc.counters(False)["lookups"] == l0
    assert (_verify(a, "schnorr", pk, msg, sig) == exp).all()
    assert kc.counters(False)["lookups"] == l0 + 16
    kb.attach()
    h = kc.counters(False)["hits"]
    assert (_verify(b, "schnorr", pk, msg, sig) == exp).all()
    assert kc.counters(False)["hits"] == h + 16
    # the creator goes first: b keeps hitting
    kc.close()
    h = kb.counters(False)["hits"]
    assert (_verify(b, "schnorr", pk, msg, sig) == exp).all()
    assert kb.counters(False)["hits"] == h + 16
    assert a._lib.kgv_keycache_counter(a._h, 0, 1) == 0
    # the last detach frees the records (2^16 Schnorr keys: about 550 MB)
    kcc = kb.on(c)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    kb.close()
    free1 = torch.cuda.mem_get_info()[0]
    kcc.close()
    free2 = torch.cuda.mem_get_info()[0]
    records = (1 << 16) * 8320
    assert free1 - free0 < records // 2 and free2 - free1 > records * 9 // 10, (free0, free1, free2)
    # kgv_keycache_clear from one context while another has calls in flight
    kc = KeyCache(a, 1 << 12, 1 << 12)
    kb = kc.on(b)
    errs = []

    def loop():
        try:
            for _ in range(20):
                assert (_verify(b, "schnorr", pk, msg, sig) == exp).all()
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = threading.Thread(target=loop, daemon=True)
    th.start()
    for _ in range(10):
        kc.clear()
    th.join(timeout=JOIN_S)
    assert not th.is_alive() and not errs, errs
    kc.clear()
    assert kb.counters(False) == dict(lookups=0, hits=0, inserts=0, evictions=0)
    kb.close()
    kc.close()


def test_cross_device_refusal(ctxs):
    import torch
    import rusty_kaspa_b200 as rk
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    d = rk.GpuContext(1)
    kc = _kc(ctxs[0], 64, 64)
    try:
        with pytest.raises(rk.KgvError, match="device"):
            kc.on(d)
    finally:
        kc.close()
        d.close()


def test_script_engine_and_replay_beside_mempool(ctxs, oracle):
    """kgv_check_scripts on engine-only spends on B finds the keys A's engine run stored; a replay window on A runs while B makes mempool
    calls, both through one cache: verdicts those of the cache-off runs"""
    from rusty_kaspa_b200 import GpuUtxoSet, Params, TransactionValidator, simgen
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_BLOCK_DTYPE
    from rusty_kaspa_b200.txbatch import build_batch
    from test_gpu_script_engine import _expected, _got, _mixed_window
    a, b = ctxs[0], ctxs[1]
    txs, ents = _mixed_window(11)
    pb, exp = _expected(oracle, txs, ents)
    kc = _kc(a)
    kb = kc.on(b)
    try:
        for c in (a, b):
            tv = TransactionValidator(c, Params(coinbase_maturity=0, storage_mass_parameter=0))
            h = kc.counters(False)["hits"]
            res = tv.validate_populated_transactions(pb, 1000, flags=2)
            assert int((res["status"] == 11).sum()) > 50
            tv.check_scripts(pb, res)
            assert _got(res) == exp
        assert kc.counters(False)["hits"] > h  # b's engine run hit a's keys

        g = simgen.FastDag(seed=9, n_keys=64, n_nonces=128, coinbase_maturity=3, mix=(0.4, 0.2, 0.2, 0.2), frac_invalid=0.1, coinbase_outputs=8)
        g.generate(24, 12)
        rb, first, pov = g.take()
        C = g.C
        arr = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
        arr["first_tx"], arr["n_txs"], arr["pov_daa_score"], arr["flags"] = first[:-1], np.diff(first), pov, 1
        fk, fe, mtxs, _ = _funded(90, 200)
        mb = build_batch(mtxs)
        prm = Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)

        def replay(c):
            rp = DagReplayer(c, Params(coinbase_maturity=3, storage_mass_parameter=C), 1 << 13)
            got, acc = rp.replay_window(rb, arr, want_accept=True)
            out = (got["status"].copy(), got["script_err"].copy(), acc.copy(), rp.us.digest())
            rp.close()
            return out

        def mempool(c):
            us = GpuUtxoSet(c, 1 << 12)
            ae, ab = simgen.entries_to_arrays(fe)
            us.apply_diff(add_keys36=fk, add_entries=ae, add_bytes=ab)
            r = TransactionValidator(c, prm).validate_mempool_transactions_in_utxo_context(us, mb, 10)[0]
            us.close()
            return r["status"].copy(), r["fee"].copy()
        import rusty_kaspa_b200 as rk
        ref = rk.GpuContext(0)
        try:
            want_r, want_m = replay(ref), mempool(ref)
        finally:
            ref.close()
        res, errs = {}, []

        def run(name, fn, c):
            try:
                res[name] = [fn(c) for _ in range(3)]
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        th = [threading.Thread(target=run, args=("r", replay, a), daemon=True), threading.Thread(target=run, args=("m", mempool, b), daemon=True)]
        [t.start() for t in th]
        [t.join(timeout=JOIN_S) for t in th]
        assert not any(t.is_alive() for t in th) and not errs, errs
        for got in res["r"]:
            assert all((np.asarray(x) == np.asarray(y)).all() if not isinstance(x, bytes) else x == y for x, y in zip(got, want_r))
        for got in res["m"]:
            assert (got[0] == want_m[0]).all() and (got[1] == want_m[1]).all()
        c = kc.counters(False)
        assert c["hits"] > 0 and c["inserts"] > 0, c
        g.close()
    finally:
        kb.close()
        kc.close()
