"""Maintenance of the GPU UTXO table: kgv_utxo_stats, kgv_utxo_rehash and the opt-in growth policy (kgv_utxo_set_max_load), checked against
a Python dict model of the set and against replays of the same blocks into a table that never rehashes."""
import numpy as np
import pytest

import oracle_tx
from rusty_kaspa_b200 import GpuUtxoSet, KgvError, MuHash, Params
from rusty_kaspa_b200.replay import DagReplayer, replay_blocks_array
from rusty_kaspa_b200.simgen import SimDag
from rusty_kaspa_b200.txbatch import ENTRY_DTYPE, build_batch

pytestmark = pytest.mark.gpu

INLINE_SCRIPT = 68


def _entries(rng, n):
    """n fresh (key, entry) pairs, scripts of 34 bytes (inline) or 100 bytes (overflow arena).  Returns keys (n, 36), ENTRY_DTYPE[n], arena."""
    keys = rng.integers(0, 256, size=(n, 36), dtype=np.uint8)
    ent = np.zeros(n, dtype=ENTRY_DTYPE)
    ent["amount"] = rng.integers(1, 1 << 50, size=n)
    ent["block_daa_score"] = rng.integers(0, 1 << 40, size=n)
    ent["spk_version"] = rng.integers(0, 2, size=n)
    ent["is_coinbase"] = rng.integers(0, 2, size=n)
    lens = np.where(rng.random(n) < 0.5, 34, 100).astype(np.uint32)
    ent["script_len"] = lens
    ent["script_off"] = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    arena = rng.integers(0, 256, size=int(lens.sum()) + 8, dtype=np.uint8)
    return keys, ent, arena


class Model:
    """the set as a dict: key bytes -> (amount, daa, spk_version, is_coinbase, script bytes)"""

    def __init__(self):
        self.d = {}

    def add(self, keys, ent, arena):
        for k, e in zip(keys, ent):
            o, n = int(e["script_off"]), int(e["script_len"])
            self.d[k.tobytes()] = (int(e["amount"]), int(e["block_daa_score"]), int(e["spk_version"]), int(e["is_coinbase"]), arena[o:o + n].tobytes())

    def remove(self, keys):
        for k in keys:
            self.d.pop(k.tobytes(), None)

    def arrays(self):
        """the content as apply_diff arguments"""
        items = sorted(self.d.items())
        keys = np.frombuffer(b"".join(k for k, _ in items), dtype=np.uint8).reshape(-1, 36)
        ent = np.zeros(len(items), dtype=ENTRY_DTYPE)
        arena, off = bytearray(), 0
        for i, (_, (a, daa, v, cb, s)) in enumerate(items):
            ent[i] = (a, daa, off, len(s), v, cb, 0)
            arena += s
            off += len(s)
        return keys, ent, np.frombuffer(bytes(arena) + bytes(8), dtype=np.uint8)

    def long_bytes(self):
        return sum((len(s) + 7) & ~7 for (_, _, _, _, s) in self.d.values() if len(s) > INLINE_SCRIPT)


def _check_lookups(us, model, keys, absent=None):
    """get() of `keys` (and of `absent`) against the model, field by field, script bytes included"""
    if absent is not None:
        keys = np.concatenate([keys, absent])
    found, got, scr = us.get(keys, script_stride=128)
    for i, k in enumerate(keys):
        m = model.d.get(k.tobytes())
        assert bool(found[i]) == (m is not None), i
        if m is None:
            continue
        a, daa, v, cb, s = m
        g = got[i]
        assert (int(g["amount"]), int(g["block_daa_score"]), int(g["spk_version"]), int(g["is_coinbase"])) == (a, daa, v, cb), i
        assert int(g["script_len"]) == len(s) and scr[i, :len(s)].tobytes() == s, i


def _exported(us):
    keys, ent, arena = us.export()
    out = {}
    for k, e in zip(keys, ent):
        o, n = int(e["script_off"]), int(e["script_len"])
        out[k.tobytes()] = (int(e["amount"]), int(e["block_daa_score"]), int(e["spk_version"]), int(e["is_coinbase"]), arena[o:o + n].tobytes())
    return out


def _model_digest(ctx, model, capacity):
    fresh = GpuUtxoSet(ctx, capacity)
    k, e, a = model.arrays()
    if len(k):
        fresh.apply_diff(add_keys36=k, add_entries=e, add_bytes=a)
    d = fresh.digest()
    fresh.close()
    return d


def test_churn_then_rehash_restores_the_table(gpu_ctx):
    cap = 1 << 14
    rng = np.random.default_rng(101)
    us = GpuUtxoSet(gpu_ctx, cap)
    model = Model()
    k, e, a = _entries(rng, 4096)
    us.apply_diff(add_keys36=k, add_entries=e, add_bytes=a)
    model.add(k, e, a)
    fresh = us.stats()
    assert fresh["capacity_slots"] == cap and fresh["live"] == 4096 and fresh["empty"] == cap - 4096 and fresh["tombstones"] == 0
    assert fresh["overflow_used"] == fresh["overflow_live"] == model.long_bytes()
    # churn: every batch erases 2048 live keys and inserts 2048 new ones.  The plain table is churned until fewer than 10 % of its slots
    # are EMPTY (churned on for 5x the capacity, one batch near 2x had an insert that did not report success); a twin with the policy on
    # takes the whole 5x the capacity of churn and never loses an entry
    pol = GpuUtxoSet(gpu_ctx, cap)
    k0, e0, a0 = model.arrays()
    pol.apply_diff(add_keys36=k0, add_entries=e0, add_bytes=a0)
    pol.set_max_load(500)
    pm = Model()
    pm.d = dict(model.d)
    live = list(model.d.keys())
    churning = True
    for step in range(40):
        idx = rng.choice(len(live), size=2048, replace=False)
        rem = np.frombuffer(b"".join(live[i] for i in idx), dtype=np.uint8).reshape(-1, 36)
        k, e, a = _entries(rng, 2048)
        if churning:
            rs, st = us.apply_diff(rem_keys36=rem, add_keys36=k, add_entries=e, add_bytes=a)
            assert (rs == 1).all() and (st == 1).all(), (step, np.unique(st, return_counts=True), us.stats())
            model.remove(rem)
            model.add(k, e, a)
            churning = us.stats()["empty"] >= cap // 10
        rs, st = pol.apply_diff(rem_keys36=rem, add_keys36=k, add_entries=e, add_bytes=a)
        assert (rs == 1).all() and (st == 1).all(), (step, pol.stats())
        pm.remove(rem)
        pm.add(k, e, a)
        gone = set(idx.tolist())
        live = [x for i, x in enumerate(live) if i not in gone] + [x.tobytes() for x in k]
    assert not churning
    ps = pol.stats()
    assert ps["insert_failures"] == 0 and ps["rehashes"] >= 1 and ps["capacity_slots"] == cap, ps  # 25 % live: rebuilt in place, never grown
    assert ps["live"] + ps["tombstones"] <= cap // 2 and ps["live"] == 4096
    assert _exported(pol) == pm.d and pol.digest() == _model_digest(gpu_ctx, pm, cap)
    pol.close()
    before = us.stats()
    assert before["live"] == len(model.d) == 4096 and before["insert_failures"] == 0
    assert before["empty"] < cap // 10, before
    assert before["tombstones"] + before["empty"] + before["live"] == cap
    assert before["longest_run"] > 3 * fresh["longest_run"], (before, fresh)
    assert before["overflow_live"] == model.long_bytes() < before["overflow_used"]
    digest_before = us.digest()
    us.rehash()
    after = us.stats()
    assert after["capacity_slots"] == cap and after["rehashes"] == 1 and after["live"] == 4096
    assert after["tombstones"] == 0 and after["empty"] == cap - 4096
    assert after["overflow_used"] == after["overflow_live"] == model.long_bytes()
    assert after["longest_run"] < 4 * fresh["longest_run"] + 16, (after, fresh)
    assert after["insert_failures"] == 0
    assert us.count() == len(model.d)
    assert us.digest() == digest_before == _model_digest(gpu_ctx, model, cap)
    assert _exported(us) == model.d
    absent = rng.integers(0, 256, size=(4096, 36), dtype=np.uint8)
    keys = np.frombuffer(b"".join(model.d.keys()), dtype=np.uint8).reshape(-1, 36)
    _check_lookups(us, model, keys, absent)
    # the rebuilt table takes writes as before
    k, e, a = _entries(rng, 1000)
    us.apply_diff(rem_keys36=keys[:500], add_keys36=k, add_entries=e, add_bytes=a)
    model.remove(keys[:500]); model.add(k, e, a)
    assert us.count() == len(model.d) and us.digest() == _model_digest(gpu_ctx, model, cap)
    us.close()


def test_grow_and_shrink_keep_the_content(gpu_ctx):
    rng = np.random.default_rng(7)
    us = GpuUtxoSet(gpu_ctx, 1 << 12)
    model = Model()
    n = int(0.85 * (1 << 12))
    k, e, a = _entries(rng, n)
    us.apply_diff(add_keys36=k, add_entries=e, add_bytes=a)
    model.add(k, e, a)
    d0 = us.digest()
    for cap in (1 << 14, 1 << 12):
        us.rehash(cap)
        s = us.stats()
        assert s["capacity_slots"] == cap and s["live"] == n and s["empty"] == cap - n and s["tombstones"] == 0
        assert s["overflow_used"] == model.long_bytes()
        assert us.digest() == d0 and us.count() == n and _exported(us) == model.d
        _check_lookups(us, model, k, rng.integers(0, 256, size=(512, 36), dtype=np.uint8))
    s0 = us.stats()
    for cap in (1 << 11, 1024, n):  # n rounds up to 4096 > n: allowed
        if cap < n:
            with pytest.raises(KgvError, match=r"\(-1\)"):
                us.rehash(cap)
            assert us.stats() == s0 and us.digest() == d0
        else:
            us.rehash(cap)
            assert us.stats()["capacity_slots"] == 1 << 12 and us.digest() == d0
    us.close()


def _view_ops(ctx, rng, rehash):
    """a base and a view layer holding FULL, FULLH, REMOVED and TOMB slots; `rehash` rebuilds base and view in between.  Returns the base
    digest after commit, and checks the composed view against the model after every step."""
    base = GpuUtxoSet(ctx, 1 << 12)
    bm = Model()
    k, e, a = _entries(rng, 1500)
    base.apply_diff(add_keys36=k, add_entries=e, add_bytes=a)
    bm.add(k, e, a)
    view = base.compose(1 << 11)
    comp = Model()
    comp.d = dict(bm.d)
    # REMOVED: erase 300 base entries through the view
    view.apply_diff(rem_keys36=k[:300])
    comp.remove(k[:300])
    # FULLH: re-add 100 of them and overwrite 100 other base entries
    k2, e2, a2 = _entries(rng, 200)
    k2 = np.concatenate([k[:100], k[300:400]])
    view.apply_diff(add_keys36=k2, add_entries=e2, add_bytes=a2)
    comp.add(k2, e2, a2)
    # FULL, then TOMB: 400 own entries, 150 of them erased again
    k3, e3, a3 = _entries(rng, 400)
    view.apply_diff(add_keys36=k3, add_entries=e3, add_bytes=a3)
    comp.add(k3, e3, a3)
    view.apply_diff(rem_keys36=k3[:150])
    comp.remove(k3[:150])
    probe = np.concatenate([k, k3, rng.integers(0, 256, size=(256, 36), dtype=np.uint8)])
    _check_lookups(view, comp, probe)
    vs = view.stats()
    assert vs["live"] == 300 + 100 + 250 and vs["tombstones"] == 150, vs  # markers count as the layer's entries
    if rehash:
        base.rehash(1 << 13)
        _check_lookups(view, comp, probe)
        _check_lookups(base, bm, k)
        view.rehash()
        s = view.stats()
        assert s["tombstones"] == 0 and s["live"] == vs["live"] and s["empty"] == s["capacity_slots"] - vs["live"] and s["rehashes"] == 1
        _check_lookups(view, comp, probe)
    view.commit()
    d = base.digest()
    assert base.count() == len(comp.d) and d == _model_digest(ctx, comp, 1 << 13)
    _check_lookups(base, comp, probe)
    view.close(); base.close()
    return d


def test_views_survive_rehash_of_base_and_layer(gpu_ctx):
    d_plain = _view_ops(gpu_ctx, np.random.default_rng(3), rehash=False)
    d_rehashed = _view_ops(gpu_ctx, np.random.default_rng(3), rehash=True)
    assert d_plain == d_rehashed


def _sim_blocks():
    dag = SimDag(seed=31, n_keys=64, n_nonces=128, mix=(0.4, 0.2, 0.2, 0.2), frac_invalid=0.12, coinbase_maturity=2, coinbase_outputs=6)
    return dag, [dag.make_block(20) for _ in range(36)]


def _windows(blocks, size=12):
    for w in range(0, len(blocks), size):
        txs, ranges = [], []
        for blk in blocks[w:w + size]:
            ranges.append((len(txs), len(blk[0]), blk[1], 1))
            txs.extend(blk[0])
        yield build_batch(txs), replay_blocks_array(ranges), list(range(len(ranges) + 1))


def test_replay_with_growth_policy_matches_the_oracle_and_a_large_table(gpu_ctx, oracle):
    dag, blocks = _sim_blocks()
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    ost = oracle_tx.State(oracle)
    op = oracle_tx.params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    exp = []
    for txs, pov in blocks:
        b = build_batch(txs)
        r = ost.validate(b, pov, 0, op, threads=2)
        exp.append(r)
        ost.accept(b, ((r["status"] == 0) | (r["status"] == 12)).astype(np.uint8), pov)
        ost.commit()
    small = DagReplayer(gpu_ctx, prm, 1 << 10, max_load=500)
    large = DagReplayer(gpu_ctx, prm, 1 << 14)
    got, n_grown_windows, at = [], 0, 0
    for b, arr, groups in _windows(blocks):
        before = small.us.stats()["rehashes"]
        rs, acs = small.replay_window(b, arr, want_accept=True)
        ms = small.replay_muhash(groups)
        rl, acl = large.replay_window(b, arr, want_accept=True)
        ml = large.replay_muhash(groups)
        assert (rs == rl).all() and (acs == acl).all()
        assert (ms == ml).all()
        n_grown_windows += small.us.stats()["rehashes"] > before
        for i in range(len(arr)):
            got.append(rs[arr[i]["first_tx"]:arr[i]["first_tx"] + arr[i]["n_txs"]])
        at += len(arr)
    for e, g in zip(exp, got):
        assert (g["status"] == e["status"]).all() and (g["script_err"] == e["script_err"]).all()
        ok = e["status"] == 0
        assert (g["fee"][ok] == e["fee"][ok]).all()
    assert small.us.count() == large.us.count() == ost.count()
    assert small.us.digest() == large.us.digest() == ost.digest()
    s = small.us.stats()
    assert s["rehashes"] >= 1 and n_grown_windows >= 1 and s["insert_failures"] == 0 and s["capacity_slots"] > 1 << 10, s
    assert s["live"] + s["tombstones"] <= s["capacity_slots"] // 2
    small.close(); large.close(); ost.close()


def test_explicit_rehash_between_windows_changes_nothing(gpu_ctx):
    dag, blocks = _sim_blocks()
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    plain = DagReplayer(gpu_ctx, prm, 1 << 12)
    rh = DagReplayer(gpu_ctx, prm, 1 << 12)
    for wi, (b, arr, groups) in enumerate(_windows(blocks)):
        r1, a1 = plain.replay_window(b, arr, want_accept=True)
        m1 = plain.replay_muhash(groups)
        r2, a2 = rh.replay_window(b, arr, want_accept=True)
        m2 = rh.replay_muhash(groups)
        assert (r1 == r2).all() and (a1 == a2).all() and (m1 == m2).all()
        rh.us.rehash((1 << 13) if wi == 1 else 0)
        # the window kgv_replay_muhash refers to ends with the rehash
        with pytest.raises(KgvError):
            rh.replay_muhash(groups)
    assert rh.us.stats()["rehashes"] == 3 and rh.us.stats()["capacity_slots"] == 1 << 13
    assert plain.us.count() == rh.us.count() and plain.us.digest() == rh.us.digest()
    assert MuHash.of_utxo_set(gpu_ctx, plain.us).finalize() == MuHash.of_utxo_set(gpu_ctx, rh.us).finalize()
    plain.close(); rh.close()


def test_policy_stays_off_unless_set(gpu_ctx):
    dag, blocks = _sim_blocks()
    prm = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
    r = DagReplayer(gpu_ctx, prm, 1 << 10)
    for b, arr, _ in _windows(blocks):
        r.replay_window(b, arr)
    s = r.us.stats()
    assert s["rehashes"] == 0 and s["capacity_slots"] == 1 << 10, s
    with pytest.raises(KgvError, match=r"\(-1\)"):
        r.us.set_max_load(901)
    r.close()
