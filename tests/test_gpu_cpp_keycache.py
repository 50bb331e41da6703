"""kgv::KeyCache of the C++ host mirror (include/kgv.hpp), driven by tests/cpp/keycache_mirror_test.cpp: Schnorr and ECDSA batches verified
cold and warm through the cache, after clear() and after the cache is gone, compared with the Python mirror's verdicts without a cache
and with the CPU oracle; the counters show the warm pass found every key."""
import os
import subprocess

import numpy as np
import pytest

from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.gpu


def test_cpp_keycache(tmp_path, gpu_ctx, oracle):
    binary = str(tmp_path / "keycache_mirror_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", binary, os.path.join(HERE, "cpp", "keycache_mirror_test.cpp"), "-L" + os.path.join(ROOT, "rusty_kaspa_b200"),
                    "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    spk, smsg, ssig, _ = W.schnorr_triples(200, seed=31, n_keys=20, n_nonces=64, frac_bitflip=0.05, frac_adversarial=0.05)
    epk, emsg, esig, _ = W.ecdsa_triples(200, seed=31, n_keys=20, n_nonces=64, frac_bitflip=0.05, frac_adversarial=0.05)
    for name, a in (("s_pk", spk), ("s_msg", smsg), ("s_sig", ssig), ("e_pk", epk), ("e_msg", emsg), ("e_sig", esig)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    out = subprocess.run([binary, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    rows = {l.split()[0] + ("" if l.split()[0] not in ("counters",) else l.split()[1]): [int(x) for x in l.split()[1:]] for l in out.stdout.splitlines() if l}
    s_py, e_py = gpu_ctx.verify_schnorr_batch(spk, smsg, ssig), gpu_ctx.verify_ecdsa_batch(epk, emsg, esig)
    assert (s_py == oracle_schnorr_batch(oracle, spk, smsg, ssig)).all() and (e_py == oracle_ecdsa_batch(oracle, epk, emsg, esig)).all()
    for tag in ("schnorr_cold", "schnorr_warm", "schnorr_cleared", "schnorr_detached"):
        assert rows[tag] == s_py.tolist(), tag
    for tag in ("ecdsa_cold", "ecdsa_warm"):
        assert rows[tag] == e_py.tolist(), tag
    for kind, pk in ((0, spk), (1, epk)):
        _, lookups, hits, inserts, evictions = rows["counters%d" % kind]
        assert lookups == 400 and hits == 200 and inserts == len(np.unique(pk, axis=0)) and evictions == 0
    assert rows["cleared"] == [200, 0]
