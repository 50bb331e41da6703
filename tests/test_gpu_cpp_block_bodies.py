"""kgv::BlockBodyProcessor of the C++ host mirror (include/kgv.hpp) driven by tests/cpp/block_body_mirror_test.cpp on dumped blocks: every
printed verdict, mass and root is compared with the CPU restatement of the reference's body rules."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import oracle_body as ob  # noqa: E402
import oracle_isolation as oi  # noqa: E402
import test_gpu_block_bodies as tb  # noqa: E402

pytestmark = pytest.mark.gpu


def test_cpp_block_body_processor(tmp_path):
    binary = str(tmp_path / "block_body_mirror_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", binary, os.path.join(HERE, "cpp", "block_body_mirror_test.cpp"), "-L" + os.path.join(ROOT, "rusty_kaspa_b200"),
                    "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    rng = np.random.default_rng(21)
    blocks = [tb.make_block(rng, 6)] + [tb._violating_block(rng, [r]) for r in tb.RULES] + [c[1] for c in ob.reference_example_blocks()]
    batch, first, h = tb.layout(blocks)
    d = str(tmp_path)
    for name, arr in (("txs", batch.txs), ("inputs", batch.inputs), ("outputs", batch.outputs), ("arena", batch.arena), ("blocks", first), ("headers", h)):
        arr.tofile(os.path.join(d, name + ".bin"))
    out = subprocess.run([binary, d, str(tb.MAX_BLOCK_MASS)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.split("\n") if l]
    assert lines[-1] == ["threw"]
    rules = oi.mainnet_rules()
    for tag, isolation_only in (("iso", True), ("ctx", False)):
        got = [l for l in lines if l[0] == tag]
        exp = ob.ok_validate_bodies(blocks, rules, tb.MAX_BLOCK_MASS, tb.MAX_PAYLOAD, isolation_only)
        assert len(got) == len(blocks)
        for k, (l, (verdict, masses)) in enumerate(zip(got, exp)):
            assert [int(x) for x in l[1:10]] == [verdict[f] for f in ("status", "index", "tx_status", "fail_input", "a", "b")] + list(masses), (tag, k, l, verdict)
            if tag == "ctx":
                assert l[10] == ob.calc_hash_merkle_root(blocks[k]["transactions"]).hex()
    assert {int(l[1]) for l in lines if l[0] == "ctx"} >= set(range(2, 16)) - {6, 7}
