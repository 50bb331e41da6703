"""kgv::HeaderProcessor of the C++ host mirror (include/kgv.hpp), driven by tests/cpp/header_mirror_test.cpp on the 1 060-transaction fixture's
headers: the same verdicts, levels and hashes as the Python binding, and the hashes the reference stored."""
import os
import subprocess

import numpy as np
import pytest

import oracle_header as oh
from rusty_kaspa_b200.headers import HeaderBatch, validate_headers_in_isolation

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_mirror_prints_the_same_verdicts(gpu_ctx, tmp_path):
    exe, libdir = str(tmp_path / "header_mirror_test"), os.path.join(ROOT, "rusty_kaspa_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "cpp", "header_mirror_test.cpp"), "-L" + libdir, "-l:libkgv.so",
                    "-Wl,-rpath," + libdir], check=True)
    params, hdrs = oh.fixture_headers(oh.FIXTURES[0])
    # a few headers that fail earlier rules, next to the fixture's
    hdrs = hdrs + [dict(hdrs[3], version=7), dict(hdrs[4], parents_by_level=[[]]), dict(hdrs[5], timestamp=2**63), dict(hdrs[6], parents_by_level=[])]
    b = HeaderBatch.from_dicts(hdrs)
    d = str(tmp_path)
    for name, arr in (("headers", b.headers), ("lens", b.level_len), ("parents", b.parents)):
        np.ascontiguousarray(arr).tofile(os.path.join(d, name + ".bin"))
    rules = oh.fixture_rules(params, skip_pow=False, now_ms=2**62)
    res, hh, _ = validate_headers_in_isolation(gpu_ctx, b, rules, want_hash=True)
    out = subprocess.run([exe, d, str(rules.now_ms), str(rules.max_block_parents), str(rules.max_block_level), str(rules.timestamp_deviation_tolerance)],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.strip().splitlines()
    want = ["%d %d %d %d %d %s" % (r["status"], r["level"], r["pow_passed"], r["a"], r["b"], hh[i].tobytes().hex()) for i, r in enumerate(res)]
    assert lines[:len(res)] == want
    assert lines[len(res)] == " ".join(x.tobytes().hex() for x in hh)
    assert [bytes.fromhex(x) for x in lines[len(res)].split()[:266]] == [h["hash"] for h in hdrs[:266]]
    assert sorted(set(res["status"].tolist())) == [1, 2, 3, 6]
