"""kgv::KeyCache of the C++ host mirror (include/kgv.hpp) shared by two kgv::Contexts, driven by tests/cpp/shared_keycache_test.cpp: two
std::threads, each on its own kgv::TransactionValidator, validate one populated batch at once through one key cache.  Every verdict
equals the serial run's and the CPU oracle's, and the shared counters show the two contexts hitting each other's keys."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
R = 6

pytestmark = pytest.mark.gpu


def test_cpp_shared_keycache(tmp_path, oracle):
    import oracle_tx
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.txbatch import build_batch
    binary = str(tmp_path / "shared_keycache_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-o", binary, os.path.join(HERE, "cpp", "shared_keycache_test.cpp"),
                    "-L" + os.path.join(ROOT, "rusty_kaspa_b200"), "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    fk, fe, txs = simgen.funded_window(120, seed=5, n_keys=24, n_nonces=64, mix=(0.4, 0.2, 0.2, 0.2))
    ents, k = [], 0
    for t in txs:
        ents.append(list(fe[k:k + len(t["inputs"])]))
        k += len(t["inputs"])
    ss = txs[9]["inputs"][0]["sigscript"]
    txs[9]["inputs"][0]["sigscript"] = ss[:20] + bytes([ss[20] ^ 4]) + ss[21:]
    b = build_batch(txs, ents)
    for name, arr in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", b.entries), ("arena", b.arena)):
        arr.tofile(str(tmp_path / (name + ".bin")))
    out = subprocess.run([binary, str(tmp_path), str(R), str(simgen.DEFAULT_STORAGE_MASS_PARAMETER)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    lines = [l.split() for l in out.stdout.splitlines() if l]
    serial = [l[1:] for l in lines if l[0] == "serial"]
    threads = [l for l in lines if l[0] == "thread"]
    counters = {int(l[1]): [int(x) for x in l[2:]] for l in lines if l[0] == "counters"}
    assert len(serial) == 2 and serial[0] == serial[1]
    assert len(threads) == 2 * R and all(l[2:] == serial[0] for l in threads)
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    want = []
    for i in range(len(txs)):
        e = oracle_tx.validate_populated(oracle, b, i, 10, 0, op)
        want.append((int(e["status"]), int(e["fee"])))
    got = [tuple(int(x) for x in v.split(":")) for v in serial[0]]
    assert [g[0] for g in got] == [w[0] for w in want] and want[9][0] != 0
    assert all(g[1] == w[1] for g, w in zip(got, want) if w[0] == 0)
    for e in (0, 1):
        lookups, hits, inserts, evictions = counters[e]
        # 2 R calls of the same keys through one cache: at most the two first ones miss
        assert evictions == 0 and 0 < inserts and lookups - hits <= 2 * lookups // (2 * R), counters[e]
