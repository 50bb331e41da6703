"""kgv::UtxoSet of the C++ host mirror (include/kgv.hpp) shared by two kgv::Contexts, driven by tests/cpp/shared_utxo_mirror_test.cpp: a
writer thread replays and commits windows on one context while a reader thread validates a mempool batch against the set through a
kgv::TransactionValidator of the other.  The scenario is tests/test_gpu_shared_utxo.py's; every verdict vector the reader prints must be
one committed version's from its serial run, versions never go back, a call that began after commit c sees version c or later, and the
handshake makes every version appear."""
import os
import subprocess

import numpy as np
import pytest

from rusty_kaspa_b200.replay import replay_blocks_array
from rusty_kaspa_b200.txbatch import build_batch
from rusty_kaspa_b200.validator import RESULT_DTYPE
from test_gpu_shared_utxo import K, Scenario, serial_run

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.gpu


def _dump(prefix, batch):
    for name, a in (("txs", batch.txs), ("inputs", batch.inputs), ("outputs", batch.outputs), ("arena", batch.arena)):
        np.ascontiguousarray(a).tofile(prefix + "_" + name + ".bin")


def test_cpp_shared_utxo(tmp_path, gpu_ctx):
    binary = str(tmp_path / "shared_utxo_mirror_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-o", binary, os.path.join(HERE, "cpp", "shared_utxo_mirror_test.cpp"),
                    "-L" + os.path.join(ROOT, "rusty_kaspa_b200"), "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    scn = Scenario()
    versions, results, _ = serial_run(scn, gpu_ctx)
    for k, blocks in enumerate(scn.windows):
        all_txs, ranges = [], []
        for txs, pov in blocks:
            ranges.append((len(all_txs), len(txs), pov, 1))  # REPLAY_ACCEPT_COINBASE, as DagReplayer.replay_windowed
            all_txs.extend(txs)
        _dump(str(tmp_path / ("w%d" % k)), build_batch(all_txs))
        replay_blocks_array(ranges).tofile(str(tmp_path / ("w%d_blocks.bin" % k)))
    _dump(str(tmp_path / "probe"), scn.probe)
    out = subprocess.run([binary, str(tmp_path), str(K), str(scn.virtual_daa), str(scn.params.coinbase_maturity), str(scn.params.storage_mass_parameter)],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    status = RESULT_DTYPE["status"]
    by_verdict = {tuple(np.frombuffer(v[1], dtype=status).tolist()): i for i, v in enumerate(versions)}
    windows, seen = {}, []
    for line in out.stdout.splitlines():
        f = line.split()
        if f[0] == "window":
            windows[int(f[1])] = [int(x) for x in f[2:]]
        elif f[0] == "read":
            v = by_verdict.get(tuple(int(x) for x in f[2:]))
            assert v is not None, "a result matches no committed version (a torn read)"
            seen.append((v, int(f[1])))
    for k in range(K):
        assert windows[k] == np.concatenate(results[k])["status"].tolist(), "replay of window %d differs from the serial run" % k
    vs = [v for v, _ in seen]
    assert all(a <= b for a, b in zip(vs, vs[1:])), "versions went back"
    assert all(v >= began for v, began in seen), "a call that began after a commit saw an older version"
    assert set(vs) == set(range(K + 1))
