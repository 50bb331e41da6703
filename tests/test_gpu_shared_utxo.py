"""One GPU UTXO set shared by several contexts (include/kgv.h, Threading): a writer context replays windows into a view over the set and
commits them, while reader contexts look entries up and validate mempool transactions against the committed set.

Every window spends outputs of the ones before it, so each committed version v = 0..K of the set gives its own lookup found-mask and its own
mempool verdicts.  A serial run on one context records them; every result a concurrent reader gets must then be exactly one version's
(no torn reads), versions never go back within a reader, and a call that began after commit c sees version c or a later one."""
import struct
import threading
import time

import numpy as np
import pytest

from rusty_kaspa_b200 import GpuContext, GpuUtxoSet, MuHash, Params, TransactionValidator
from rusty_kaspa_b200.replay import DagReplayer
from rusty_kaspa_b200.simgen import SimDag, tx_id
from rusty_kaspa_b200.txbatch import build_batch

pytestmark = pytest.mark.gpu

K = 6              # windows
BLOCKS = 3         # blocks per window
TXS = 12           # transactions per block
JOIN_S = 300       # a thread or handshake that takes longer has hung: the test fails instead of waiting for ever


def _key(txid, index):
    return bytes(txid) + struct.pack("<I", index)


class Scenario:
    """K windows of a seeded chain.  After window k is generated, one of its transaction outputs is held back from the generator (never
    spent later) and a mempool transaction spending it is signed: that transaction is missing its outpoint in versions <= k and valid
    from version k + 1 on.  The lookup probe is every outpoint the windows create, so outputs created in one window and spent in a later
    one exist only in the versions between."""

    def __init__(self, seed=23):
        dag = SimDag(seed=seed, n_keys=64, n_nonces=128, coinbase_maturity=2, coinbase_outputs=4)
        self.params = Params(coinbase_maturity=2, storage_mass_parameter=dag.C)
        self.windows, keys, probe_txs = [], [], []
        for _ in range(K):
            blocks = [dag.make_block(TXS) for _ in range(BLOCKS)]
            self.windows.append(blocks)
            for txs, _ in blocks:
                for tx in txs:
                    tid = tx_id(tx)
                    keys += [_key(tid, i) for i in range(len(tx["outputs"]))]
            held = next(u for u in reversed(dag.utxos) if not u["coinbase"])
            dag.utxos.remove(held)
            rest, dag.utxos = dag.utxos, [held]
            tx = dag._make_tx(dag.daa + 1, set(), [])
            dag.utxos = rest
            assert tx is not None
            probe_txs.append(tx)
        self.keys = np.frombuffer(b"".join(keys), dtype=np.uint8).reshape(-1, 36)
        self.probe = build_batch(probe_txs)
        self.virtual_daa = dag.daa + 100


def lookup_mask(us, keys):
    found, _, _ = us.get(keys, script_stride=128)
    return found.tobytes()


def mempool_verdicts(tv, us, scn):
    res = tv.validate_mempool_transactions_in_utxo_context(us, scn.probe, scn.virtual_daa)[0]
    return res["status"].tobytes()


class Writer:
    """Context A: a DagReplayer whose table is a view over the committed set."""

    def __init__(self, ctx, scn, capacity=1 << 13, view_capacity=1 << 12, max_load=None):
        self.rep = DagReplayer(ctx, scn.params, capacity, max_load=max_load)
        self.base = self.rep.us
        self.view = self.base.compose(view_capacity)
        self.rep.us = self.view

    def replay(self, blocks):
        return self.rep.replay_windowed(blocks)

    def commit(self):
        self.view.commit()

    def close(self):
        self.view.close()
        self.base.close()


def serial_run(scn, ctx, capacity=1 << 13, max_load=None):
    """versions[v] = (found-mask, mempool verdicts) of committed version v; results[k] = the replay results of window k"""
    w = Writer(ctx, scn, capacity, max_load=max_load)
    tv = TransactionValidator(ctx, scn.params)
    versions, results = [], []
    for k in range(K + 1):
        versions.append((lookup_mask(w.base, scn.keys), mempool_verdicts(tv, w.base, scn)))
        if k < K:
            results.append(w.replay(scn.windows[k]))
            w.commit()
    final = (w.base.count(), w.base.digest(), MuHash.of_utxo_set(ctx, w.base).finalize())
    w.close()
    masks, verdicts = [v[0] for v in versions], [v[1] for v in versions]
    assert len(set(masks)) == K + 1 and len(set(verdicts)) == K + 1, "every version must give its own answer"
    return versions, results, final


@pytest.fixture(scope="module")
def scn():
    return Scenario()


@pytest.fixture(scope="module")
def serial(scn, gpu_ctx):
    return serial_run(scn, gpu_ctx)


class Reader(threading.Thread):
    """Looks up the probe keys and validates the mempool probe on the base, through its own context, until told to stop.  Records, per call,
    the version its result equals and the commits completed before the call began."""

    def __init__(self, ctx, base, scn, versions, board):
        super().__init__(daemon=True)
        self.ctx, self.us, self.scn, self.board = ctx, base.on(ctx), scn, board
        self.tv = TransactionValidator(ctx, scn.params)
        self.by_mask = {v[0]: i for i, v in enumerate(versions)}
        self.by_verdict = {v[1]: i for i, v in enumerate(versions)}
        self.seen, self.errors, self.done_after = [], [], -1

    def run(self):
        try:
            n = 0
            while not self.board.stop.is_set():
                began = self.board.commits
                if n % 2 == 0:
                    v = self.by_mask.get(lookup_mask(self.us, self.scn.keys))
                else:
                    v = self.by_verdict.get(mempool_verdicts(self.tv, self.us, self.scn))
                self.seen.append((v, began, n % 2))
                self.done_after = began
                n += 1
        except Exception as e:  # pragma: no cover - reported by the test
            self.errors.append(repr(e))

    def check(self):
        assert not self.errors, self.errors
        assert self.seen, "the reader made no call"
        vs = [v for v, _, _ in self.seen]
        assert None not in vs, "a result matches no committed version (a torn read)"
        assert all(a <= b for a, b in zip(vs, vs[1:])), "versions went back within a reader"
        assert all(v >= began for v, began, _ in self.seen), "a call that began after a commit saw an older version"
        return set(vs)


class Board:
    def __init__(self):
        self.commits = 0
        self.stop = threading.Event()


def wait_for(cond, what):
    t0 = time.monotonic()
    while not cond():
        if time.monotonic() - t0 > JOIN_S:
            raise AssertionError("timed out waiting for " + what)
        time.sleep(0.0005)


def concurrent_run(scn, serial, handshake, rehash=False, capacity=1 << 13, max_load=None):
    versions, results, final = serial
    ctx_a, ctx_b, ctx_c = GpuContext(0), GpuContext(0), GpuContext(0)
    w = Writer(ctx_a, scn, capacity, max_load=max_load)
    board = Board()
    readers = [Reader(c, w.base, scn, versions, board) for c in (ctx_b, ctx_c)]
    try:
        for r in readers:
            r.start()
        if handshake:
            wait_for(lambda: all(r.done_after >= 0 for r in readers), "the readers' first calls")
        for k in range(K):
            got = w.replay(scn.windows[k])
            for a, e in zip(got, results[k]):
                assert a.tobytes() == e.tobytes(), "replay results differ from the serial run, window %d" % k
            w.commit()
            if rehash:
                cap = w.base.stats()["capacity_slots"]
                w.base.rehash(2 * cap)
                w.base.rehash(0)
            board.commits = k + 1
            if handshake:
                wait_for(lambda: all(r.done_after >= k + 1 for r in readers), "a read after commit %d" % (k + 1))
        if not handshake:
            wait_for(lambda: all(r.done_after >= K for r in readers), "a read after the last commit")
    finally:
        board.stop.set()
        for r in readers:
            r.join(JOIN_S)
    assert not any(r.is_alive() for r in readers), "a reader thread hung"
    seen = set()
    for r in readers:
        seen |= r.check()
        assert {m for _, _, m in r.seen} == {0, 1}, "a reader made only one kind of call"
    got_final = (w.base.count(), w.base.digest(), MuHash.of_utxo_set(ctx_a, w.base).finalize())
    assert got_final == final, "the committed set differs from the serial run's"
    w.close()
    for c in (ctx_a, ctx_b, ctx_c):
        c.close()
    return seen


def test_every_version_seen_with_handshake(scn, serial):
    seen = concurrent_run(scn, serial, handshake=True)
    assert seen == set(range(K + 1))


def test_free_running_readers(scn, serial):
    concurrent_run(scn, serial, handshake=False)


def test_rehash_between_commits_under_readers(scn, serial):
    seen = concurrent_run(scn, serial, handshake=True, rehash=True)
    assert seen == set(range(K + 1))


def test_growth_inside_commits_under_readers(scn, gpu_ctx):
    # a small table with the growth policy on: commits rehash the base while the readers read it
    small = serial_run(scn, gpu_ctx, capacity=1 << 10, max_load=100)
    seen = concurrent_run(scn, small, handshake=True, capacity=1 << 10, max_load=100)
    assert seen == set(range(K + 1))


def test_replay_beside_mempool(scn, serial):
    """A replay into the view on A runs while B validates mempool transactions against the base: B is not held up by the replay (it
    writes the view and only reads the base), and sees the version before the window's commit."""
    versions, results, final = serial
    ctx_a, ctx_b = GpuContext(0), GpuContext(0)
    w = Writer(ctx_a, scn)
    tv_b = TransactionValidator(ctx_b, scn.params)
    base_b = w.base.on(ctx_b)
    overlapped = 0
    try:
        for k in range(K):
            out, err = {}, []
            replaying = threading.Event()

            def replay():
                try:
                    replaying.set()
                    out["res"] = w.replay(scn.windows[k])
                except Exception as e:  # pragma: no cover - reported below
                    err.append(repr(e))

            t = threading.Thread(target=replay, daemon=True)
            t.start()
            replaying.wait(JOIN_S)
            calls = 0
            while t.is_alive() or calls == 0:
                assert mempool_verdicts(tv_b, base_b, scn) == versions[k][1], "window %d" % k
                calls += 1
            t.join(JOIN_S)
            assert not t.is_alive() and not err, err
            overlapped += calls > 1
            for a, e in zip(out["res"], results[k]):
                assert a.tobytes() == e.tobytes(), "replay results differ from the serial run, window %d" % k
            w.commit()
        assert mempool_verdicts(tv_b, base_b, scn) == versions[K][1]
        assert overlapped > 0, "no mempool call ran during a replay"
    finally:
        w.close()
        ctx_a.close()
        ctx_b.close()

