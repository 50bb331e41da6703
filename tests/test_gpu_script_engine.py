"""The device script engine (kgv_check_scripts, and the table-backed calls that run it on the spends the fast path declines) against the
host engine (kgv_check_scripts_host, pinned by the reference corpus in tests/test_host_vm.py): the corpus, the mainnet KATs and random
scripts with host and with device pointers, mixed windows through kgv_validate_txs / validate_transactions_with_muhash_in_parallel /
kgv_validate_mempool_txs / kgv_replay_window, and a SigCache run."""
import copy
import ctypes
import hashlib
import random

import numpy as np
import pytest

from golden_util import entry_from_json, load, tx_from_json
from rusty_kaspa_b200 import MuHash, Params, TransactionValidator
from rusty_kaspa_b200.simgen import SUBNET_COINBASE, SUBNET_NATIVE, SimDag, sighash_all
from rusty_kaspa_b200.txbatch import build_batch
from rusty_kaspa_b200.validator import RESULT_DTYPE, SigCache, script_execute
from rusty_kaspa_b200.verifier import _KgvTxBatch, _c_batch
from test_gpu_host_vm import _custom_spends, _load_entries
from test_host_vm import oracle_verdicts, spending_tx
from test_hostsim_script import random_tx

pytestmark = pytest.mark.gpu


def _host(ctx, b, idx):
    out = np.zeros(len(idx), dtype=RESULT_DTYPE)
    cb = _c_batch(b, with_entries=True)
    ctx._check(ctx._lib.kgv_check_scripts_host(ctx._h, ctypes.byref(cb), idx.ctypes.data, len(idx), out.ctypes.data))
    return out


def _dev_host_ptrs(ctx, b, idx):
    out = np.zeros(len(idx), dtype=RESULT_DTYPE)
    cb = _c_batch(b, with_entries=True)
    ctx._check(ctx._lib.kgv_check_scripts(ctx._h, ctypes.byref(cb), idx.ctypes.data, len(idx), out.ctypes.data))
    return out


def _dev_dev_ptrs(ctx, b, idx):
    import torch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    t = {k: dev(v) for k, v in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", b.entries), ("arena", b.arena), ("idx", idx))}
    res = torch.zeros(len(idx) * 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    cb = _KgvTxBatch(t["txs"].data_ptr(), len(b.txs), t["inputs"].data_ptr(), len(b.inputs), t["outputs"].data_ptr(), len(b.outputs),
                     t["entries"].data_ptr(), t["arena"].data_ptr(), len(b.arena))
    ctx._check(ctx._lib.kgv_check_scripts(ctx._h, ctypes.byref(cb), t["idx"].data_ptr(), len(idx), res.data_ptr()))
    ctx._check(ctx._lib.kgv_synchronize(ctx._h))
    return res.cpu().numpy().view(RESULT_DTYPE)


def _same(a, b):
    for f in ("status", "script_err", "fail_input"):
        bad = np.nonzero(a[f] != b[f])[0]
        assert len(bad) == 0, (f, bad[:5], a[bad[:5]], b[bad[:5]])


def _all_three(ctx, b):
    idx = np.arange(len(b.txs), dtype=np.uint32)
    exp = _host(ctx, b, idx)
    _same(_dev_host_ptrs(ctx, b, idx), exp)
    _same(_dev_dev_ptrs(ctx, b, idx), exp)
    return exp


def test_corpus_and_kats(gpu_ctx):
    rows = [r for r in load("script_tests.json.gz")["rows"] if "builder_error" not in r]
    txs, ents = zip(*[spending_tx(bytes.fromhex(r["sigscript"]), bytes.fromhex(r["spk"])) for r in rows])
    exp = _all_three(gpu_ctx, build_batch(list(txs), list(ents)))
    assert (exp["status"] == 0).sum() > 100 and len(set(exp["script_err"].tolist())) >= 20
    txs, ents = [], []
    for c in load("check_scripts_kat.json")["cases"]:
        tx, entries = tx_from_json(c["tx"]), [entry_from_json(e) for e in c["entries"]]
        tx2 = copy.deepcopy(tx)
        tx2["inputs"].append(copy.deepcopy(tx2["inputs"][-1]))
        txs += [tx, tx2]; ents += [entries, entries + [copy.deepcopy(entries[-1])]]
    _all_three(gpu_ctx, build_batch(txs, ents))


def test_random_scripts(gpu_ctx):
    rng = random.Random(77)
    txs, ents = zip(*[random_tx(rng) for _ in range(10_000)])
    b = build_batch(list(txs), list(ents))
    exp = _all_three(gpu_ctx, b)
    assert len(set(exp["script_err"].tolist())) >= 25
    # a subset, in a scrambled order, with repeats
    idx = np.array(rng.sample(range(len(txs)), 500) * 2, dtype=np.uint32)
    _same(_dev_host_ptrs(gpu_ctx, b, idx), _host(gpu_ctx, b, idx))


def _envelope_spends(n, seed, dag):
    """P2SH data envelopes: redeem = <pk> CHECKSIG FALSE IF "kasplex" 00 <json> ENDIF"""
    rng = np.random.default_rng(seed)
    txs, ents = [], []
    for t in range(n):
        k = int(rng.integers(0, dag.keys.count))
        pk = dag.keys.xs[k]
        body = b'{"p":"krc-20","op":"mint","tick":"T%d"}' % t
        redeem = b"\x20" + pk + b"\xac\x00\x63\x07kasplex\x00\x4c" + bytes([len(body)]) + body + b"\x68"
        spk = b"\xaa\x20" + hashlib.blake2b(redeem, digest_size=32).digest() + b"\x87"
        entry = {"amount": 10**9, "spk_version": 0, "script": spk, "block_daa_score": 5, "is_coinbase": False}
        tx = {"version": 0, "inputs": [{"txid": bytes(rng.integers(0, 256, 32, dtype=np.uint8)), "index": 1, "sigscript": b"", "sequence": 0, "sig_op_count": 1}],
              "outputs": [{"value": 10**9 - 1, "spk_version": 0, "script": b"\x20" + pk + b"\xac"}], "lock_time": 0, "subnetwork_id": SUBNET_NATIVE,
              "gas": 0, "payload": b"", "mass": 0}
        msg = sighash_all(tx, [entry], 0, False)
        sig = dag._sign(k, msg if t % 5 else bytes(32), False)
        tx["inputs"][0]["sigscript"] = b"\x41" + sig + b"\x01" + (bytes([0x4C, len(redeem)]) if len(redeem) > 75 else bytes([len(redeem)])) + redeem
        txs.append(tx); ents.append([entry])
    return txs, ents


def _mixed_window(seed):
    """standard spends, the custom shapes, envelopes, a > 68-byte spk and two-input transactions whose non-standard input follows a
    failing standard one"""
    dag = SimDag(seed=seed, n_keys=32, n_nonces=64)
    txs, ents = _custom_spends(64, seed)
    t2, e2 = _envelope_spends(24, seed + 1, dag)
    txs += t2; ents += e2
    for j in range(8):  # a standard P2PK input (bad signature for even j) followed by an envelope input
        pk = dag.keys.xs[j]
        tx, e = _envelope_spends(1, 100 + j, dag)
        tx, e = tx[0], e[0]
        std_entry = {"amount": 10**9, "spk_version": 0, "script": b"\x20" + pk + b"\xac", "block_daa_score": 5, "is_coinbase": False}
        tx["inputs"].insert(0, {"txid": bytes([0xD0 + j]) * 32, "index": 0, "sigscript": b"", "sequence": 0, "sig_op_count": 1})
        ents_t = [std_entry] + e
        tx["outputs"][0]["value"] = 10**9
        msg0 = sighash_all(tx, ents_t, 0, False)
        tx["inputs"][0]["sigscript"] = b"\x41" + dag._sign(j, msg0 if j % 2 else bytes(32), False) + b"\x01"
        # the envelope input's signature is over the final tx
        ss1 = tx["inputs"][1]["sigscript"]
        redeem = ss1[66 + (2 if ss1[66] == 0x4C else 1):]
        k1 = next(i for i in range(dag.keys.count) if dag.keys.xs[i] == redeem[1:33])
        msg1 = sighash_all(tx, ents_t, 1, False)
        tx["inputs"][1]["sigscript"] = b"\x41" + dag._sign(k1, msg1, False) + b"\x01" + ss1[66:]
        txs.append(tx); ents.append(ents_t)
    # standard spends from the generator's own window
    pk = dag.keys.xs[3]
    long_spk = b"\x20" + pk + b"\xad" + b"".join(b"\x0a" + bytes([7] * 10) + b"\x75" for _ in range(8)) + b"\x51"
    entry = {"amount": 10**9, "spk_version": 0, "script": long_spk, "block_daa_score": 5, "is_coinbase": False}
    tx = {"version": 0, "inputs": [{"txid": b"\xee" * 32, "index": 3, "sigscript": b"", "sequence": 0, "sig_op_count": 1}],
          "outputs": [{"value": 10**9 - 1, "spk_version": 0, "script": b"\x20" + pk + b"\xac"}], "lock_time": 0, "subnetwork_id": SUBNET_NATIVE,
          "gas": 0, "payload": b"", "mass": 0}
    tx["inputs"][0]["sigscript"] = b"\x41" + dag._sign(3, sighash_all(tx, [entry], 0, False), False) + b"\x01"
    txs.append(tx); ents.append([entry])
    for j in range(16):  # plain P2PK spends the fast path decides
        pkj = dag.keys.xs[j]
        e = {"amount": 10**9, "spk_version": 0, "script": b"\x20" + pkj + b"\xac", "block_daa_score": 5, "is_coinbase": False}
        t = {"version": 0, "inputs": [{"txid": bytes([0x70 + j]) * 32, "index": 0, "sigscript": b"", "sequence": 0, "sig_op_count": 1}],
             "outputs": [{"value": 10**9 - 1, "spk_version": 0, "script": b"\x51"}], "lock_time": 0, "subnetwork_id": SUBNET_NATIVE, "gas": 0, "payload": b"", "mass": 0}
        t["inputs"][0]["sigscript"] = b"\x41" + dag._sign(j, sighash_all(t, [e], 0, False) if j % 3 else bytes(32), False) + b"\x01"
        txs.append(t); ents.append([e])
    return txs, ents


def _expected(oracle, txs, ents):
    pb = build_batch(txs, ents)
    exp = []
    for i, t in enumerate(txs):
        r = (0, 0, 0)
        for k in range(len(t["inputs"])):
            e = script_execute(pb, i, k, oracle_verdicts(oracle, pb))
            if e:
                r = (9 if t["inputs"][k]["sigscript"] else 10, e, k)
                break
        exp.append(r)
    return pb, exp


def _got(res):
    return [(int(r["status"]), int(r["script_err"]), int(r["fail_input"]) if r["status"] else 0) for r in res]


def test_mixed_windows_through_the_table_calls(gpu_ctx, oracle):
    from rusty_kaspa_b200 import GpuUtxoSet
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_ACCEPT_COINBASE
    txs, ents = _mixed_window(11)
    pb, exp = _expected(oracle, txs, ents)
    assert sum(1 for e in exp if e[0] == 0) > 20 and sum(1 for e in exp if e[0]) > 10
    assert any(e[0] and e[2] == 0 and len(t["inputs"]) == 2 for e, t in zip(exp, txs))
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=0, storage_mass_parameter=0))
    # kgv_check_scripts on what the fast path declines, in a populated host batch
    res = tv.validate_populated_transactions(pb, 1000, flags=2)
    n_declined = int((res["status"] == 11).sum())
    assert n_declined > 50
    tv.check_scripts(pb, res)
    assert _got(res) == exp
    # kgv_validate_txs and the MuHash of the accepted transactions
    us = GpuUtxoSet(gpu_ctx, 1 << 12)
    _load_entries(us, txs, ents)
    b = build_batch(txs)
    res, mu = tv.validate_transactions_with_muhash_in_parallel(us, b, 1000, flags=2)
    assert _got(res) == exp
    acc = (res["status"] == 0).astype(np.uint8)
    assert mu.numerator == MuHash.from_transactions(gpu_ctx, pb, acc, 1000).numerator
    # kgv_validate_mempool_txs, the first half of the entries supplied by the caller
    sup = np.zeros(len(pb.inputs), dtype=bool)
    sup[: len(sup) // 2] = True
    mres, mass, ent_out, _ = tv.validate_mempool_transactions_in_utxo_context(us, pb, 1000, supplied=sup)
    assert _got(mres) == exp
    us.close()
    # kgv_replay_window: the same spends as one block (tx 0 = coinbase)
    cb = {"version": 0, "inputs": [], "outputs": [{"value": 5, "spk_version": 0, "script": b"\x51"}], "lock_time": 0, "subnetwork_id": SUBNET_COINBASE,
          "gas": 0, "payload": b"x", "mass": 0}
    r = DagReplayer(gpu_ctx, Params(coinbase_maturity=0, storage_mass_parameter=0), 1 << 12)
    _load_entries(r.us, txs, ents)
    out = r.replay_windowed([([cb] + txs, 1000, REPLAY_ACCEPT_COINBASE)])[0]
    assert _got(out[1:]) == exp and out[0]["status"] == 12
    assert r.last_stats["n_host_vm"] == n_declined
    n_in = sum(len(t["inputs"]) for t in txs)
    assert r.us.count() == 1 + int(acc.sum()) + (n_in - sum(len(t["inputs"]) for t, a in zip(txs, acc) if a))
    r.close()


def test_sigcache_answers_the_engine_checks(gpu_ctx, oracle):
    txs, ents = _envelope_spends(40, 5, SimDag(seed=5, n_keys=32, n_nonces=64))
    pb, exp = _expected(oracle, txs, ents)
    tv = TransactionValidator(gpu_ctx, Params(coinbase_maturity=0, storage_mass_parameter=0))
    sc = SigCache(gpu_ctx, 4096)
    sc.attach()
    try:
        res1 = tv.validate_populated_transactions(pb, 1000, flags=2)
        tv.check_scripts(pb, res1)
        c1 = sc.counters()
        res2 = tv.validate_populated_transactions(pb, 1000, flags=2)
        tv.check_scripts(pb, res2)
        c2 = sc.counters()
    finally:
        sc.close()
    assert _got(res1) == exp and _got(res2) == exp
    assert c1["inserts"] >= 32 and c2["hits"] - c1["hits"] >= 32  # the second pass is answered from the cache


def test_sharded_replay_with_nonstandard_spends(oracle):
    """two contexts replay one window with kgv_set_sharding on (test_gpu_comm's set-up): the fast path's pairs are split over the ranks and
    exchanged, the declined transactions go through the device engine on every rank.  Verdicts, accept mask, UTXO count / digest and the
    window's MuHash equal the expectation from the oracle plus the host engine, applied to a table of its own."""
    import torch
    from rusty_kaspa_b200 import GpuUtxoSet
    from rusty_kaspa_b200.comm import ShardComm
    from rusty_kaspa_b200.replay import DagReplayer, REPLAY_ACCEPT_COINBASE, replay_blocks_array
    from test_gpu_comm import _contexts, _run_ranks
    txs, ents = _mixed_window(23)
    pb, exp = _expected(oracle, txs, ents)
    cb = {"version": 0, "inputs": [], "outputs": [{"value": 5, "spk_version": 0, "script": b"\x51"}], "lock_time": 0, "subnetwork_id": SUBNET_COINBASE,
          "gas": 0, "payload": b"sharded", "mass": 0}
    for t in txs:
        t["mass"] = 0  # C = 0: the storage mass the replay's context rules expect
    b = build_batch([cb] + txs)
    arr = replay_blocks_array([(0, len(txs) + 1, 1000, REPLAY_ACCEPT_COINBASE)])
    prm = Params(coinbase_maturity=0, storage_mass_parameter=0)
    n_ranks = 2
    ctxs = _contexts(n_ranks)
    # the expectation: accept what the oracle + host engine accept, on a table of its own
    acc_exp = np.array([1] + [1 if e[0] == 0 else 0 for e in exp], dtype=np.uint8)
    us = GpuUtxoSet(ctxs[0], 1 << 12)
    _load_entries(us, txs, ents)
    mu_exp = MuHash.from_transactions(ctxs[0], b, acc_exp, 1000, utxo_set=us).finalize()
    us.add_transactions(b, acc_exp, 1000)
    cnt_exp, dig_exp = us.count(), us.digest()
    us.close()
    comms = [ShardComm(ctxs[r], n_ranks, r, slice_capacity=1 << 20) for r in range(n_ranks)]
    ShardComm.connect_local(comms)
    reps = [DagReplayer(ctxs[r], prm, 1 << 12) for r in range(n_ranks)]
    for rp in reps:
        _load_entries(rp.us, txs, ents)
    if torch.cuda.device_count() < n_ranks:  # size every per-call buffer up front with an unsharded dry run (see test_gpu_comm)
        for r in range(n_ranks):
            scratch = DagReplayer(ctxs[r], prm, 1 << 12)
            _load_entries(scratch.us, txs, ents)
            scratch.replay_window(b, arr)
            scratch.close()

    def rank_body(r):
        comms[r].shard_validation(True)
        res, acc = reps[r].replay_window(b, arr, want_accept=True)
        mu = reps[r].replay_muhash([0, 1])[0]
        return res, acc, mu, reps[r].us.count(), reps[r].us.digest()
    out = _run_ranks(rank_body, n_ranks)
    for r in range(n_ranks):
        res, acc, mu, cnt, dig = out[r]
        assert _got(res[1:]) == exp and res[0]["status"] == 12, r
        assert (acc == acc_exp).all() and cnt == cnt_exp and dig == dig_exp, r
        assert MuHash(ctxs[r], mu[:384].tobytes(), mu[384:].tobytes()).finalize() == mu_exp, r
    for c in comms:
        c.close()
    for rp in reps:
        rp.close()
    for c in ctxs:
        c.close()


def test_cpp_mirror_check_scripts(tmp_path, oracle):
    """kgv::TransactionValidator::check_scripts (include/kgv.hpp) through tests/cpp/script_engine_mirror_test, built by build()"""
    import os
    import subprocess
    binary = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "script_engine_mirror_test")
    assert os.path.exists(binary), "script_engine_mirror_test missing: run __graft_entry__.build()"
    txs, ents = _mixed_window(31)
    pb, exp = _expected(oracle, txs, ents)
    d = str(tmp_path)
    for name, arr in (("txs", pb.txs), ("inputs", pb.inputs), ("outputs", pb.outputs), ("entries", pb.entries), ("arena", pb.arena)):
        arr.tofile(os.path.join(d, name + ".bin"))
    out = subprocess.run([binary, d, "1000"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.split("\n") if l.startswith("tx ")]
    assert len(lines) == len(txs)
    assert sum(1 for f in lines if int(f[1]) == 11) > 50  # declined by the fast path ...
    got = [(int(f[2]), int(f[3]), int(f[4]) if int(f[2]) else 0) for f in lines]
    assert got == exp  # ... and decided by the device engine
    for f, e, t, en in zip(lines, exp, txs, ents):  # the fee survives the engine's update
        if e[0] == 0:
            assert int(f[5]) == sum(x["amount"] for x in en) - sum(o["value"] for o in t["outputs"])
