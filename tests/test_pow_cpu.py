"""GPU-less tests of header validation in isolation: the cSHAKE256 start states, Keccak-f1600, the proof-of-work matrix known answers,
compact-bits decoding and whole headers, each in three independent places that must agree: the Python restatement (oracle_header.py),
the C restatement (tests/oracle_pow/ok_pow.c) and the host build of the device code (tests/hostsim/hostsim_pow.cpp)."""
import ctypes
import hashlib
import json
import os
import random
import re
import struct
import sys

import numpy as np
import pytest

import oracle_header as oh
from rusty_kaspa_b200.headers import HEADER_RESULT_DTYPE, HeaderBatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import derive_cshake_states as dcs  # noqa: E402

KAT = json.load(open(os.path.join(oh.GOLDEN, "pow_kat.json")))


@pytest.fixture(scope="module")
def ok():
    return oh.c_oracle()


@pytest.fixture(scope="module")
def hs():
    return oh.hostsim()


def _u16(m):
    return np.ascontiguousarray(np.array(m, dtype=np.uint16))


def _u8(m):
    return np.ascontiguousarray(np.array(m, dtype=np.uint8))


def test_device_constants_are_the_derived_states():
    src = open(os.path.join(ROOT, "rusty_kaspa_b200", "csrc", "kgv_keccak.cuh")).read()
    s = dcs.derive()
    for name, key in (("kPowHashStart", "ProofOfWorkHash"), ("kHeavyHashStart", "HeavyHash")):
        body = src[src.index(name + "[25]"):]
        words = [int(x, 16) for x in re.findall(r"0x([0-9a-f]{16})ull", body[:body.index("};")])]
        assert words == s[key], name


def test_derived_states_reproduce_the_heavy_hash_known_answer():
    k = KAT["heavy_hash"]
    assert oh.heavy_hash(k["matrix"], bytes.fromhex(k["input"])).hex() == k["expected"]


@pytest.mark.parametrize("msg_len", [0, 1, 31, 32, 80, 135])
def test_keccak_f1600_agrees_with_sha3_256(ok, hs, msg_len):
    msg = bytes(random.Random(msg_len).randrange(256) for _ in range(msg_len))
    blk = bytearray(136)
    blk[:msg_len] = msg
    blk[msg_len] ^= 0x06
    blk[135] ^= 0x80
    st = list(struct.unpack("<17Q", bytes(blk))) + [0] * 8
    want = hashlib.sha3_256(msg).digest()
    assert b"".join(w.to_bytes(8, "little") for w in dcs.keccak_f1600(list(st))[:4]) == want
    for f in (ok.ok_keccak_f1600, hs.hs_keccak_f1600):
        a = np.array(st, dtype=np.uint64)
        f(a.ctypes.data)
        assert a[:4].tobytes() == want


def test_generate_matrix_known_answer(ok, hs):
    k = KAT["generate_matrix"]
    seed, want = bytes.fromhex(k["seed"]), k["matrix"]
    m, tries = oh.generate_matrix(seed)
    assert m == want and tries == 1
    for f in (ok.ok_pow_generate, hs.hs_generate):
        out = np.zeros(4096, dtype=np.uint8)
        assert f(seed, out.ctypes.data) == 1
        assert out.reshape(64, 64).tolist() == want


def test_heavy_hash_known_answer(ok, hs):
    k = KAT["heavy_hash"]
    m = _u8(k["matrix"])
    for f in (ok.ok_pow_heavy_hash, hs.hs_heavy_hash):
        out = np.zeros(32, dtype=np.uint8)
        f(m.ctypes.data, bytes.fromhex(k["input"]), out.ctypes.data)
        assert out.tobytes().hex() == k["expected"]


@pytest.mark.parametrize("case", [c["name"] for c in KAT["compute_rank"]])
def test_compute_rank_known_answers(ok, hs, case):
    c = next(c for c in KAT["compute_rank"] if c["name"] == case)
    m = _u16(c["matrix"])
    assert oh.compute_rank(c["matrix"]) == c["rank"]
    assert ok.ok_pow_rank_u16(m.ctypes.data) == c["rank"]
    assert hs.hs_rank(m.ctypes.data) == c["rank"]


def test_rank_edge_cases_agree(ok, hs):
    rng = random.Random(5)
    cases = []
    full = [[rng.randrange(16) for _ in range(64)] for _ in range(64)]
    cases.append(full)
    for r in (1, 17, 40, 63):  # rows beyond r are combinations of the first r: rank r
        base = [[rng.randrange(16) for _ in range(64)] for _ in range(r)]
        cases.append(base + [[sum(base[(i + t) % r][c] for t in range(2)) for c in range(64)] for i in range(64 - r)])
    cases.append([[1 if c == r else 0 for c in range(64)] for r in range(64)])
    cases.append([[0] * 64 if r == 7 else list(full[r]) for r in range(64)])
    cases.append([[(r * c) % 16 for c in range(64)] for r in range(64)])
    for m in cases:
        want = oh.compute_rank(m)
        a = _u16(m)
        assert ok.ok_pow_rank_u16(a.ctypes.data) == want and hs.hs_rank(a.ctypes.data) == want


def test_generate_retries_until_full_rank(hs):
    """Matrix::generate's loop, on candidates the caller scripts: rank-deficient ones are skipped, the first full-rank one is kept."""
    full = KAT["generate_matrix"]["matrix"]
    zero = [[0] * 64 for _ in range(64)]
    dup = [list(full[1])] + [list(r) for r in full[1:]]
    assert oh.compute_rank(dup) == 63
    for cands, want_tries in (([full], 1), ([zero, full], 2), ([zero, dup, dup, full], 4)):
        arr = _u8(cands)
        out = np.zeros(4096, dtype=np.uint8)
        assert hs.hs_generate_scripted(arr.ctypes.data, len(cands), out.ctypes.data) == want_tries
        assert out.reshape(64, 64).tolist() == full


def _bits_cases():
    out = []
    for e in range(256):
        for mant in (0, 1, 0x7F, 0x80, 0x1234, 0x7FFFFF, 0x800000, 0x800001, 0xFFFFFF, 0x123456 | 0x800000):
            out.append((e << 24) | mant)
    return out


def _python_compact(bits):
    """from_compact_target_bits restated on Python integers: mantissa and exponent as math/src/lib.rs:64-79, the shift as
    math/src/uint.rs overflowing_shl (s mod 256, bits past 2^256 dropped)."""
    e = bits >> 24
    if e <= 3:
        mant, s = (bits & 0xFFFFFF) >> (8 * (3 - e)), 0
    else:
        mant, s = bits & 0xFFFFFF, 8 * (e - 3)
    if mant > 0x7FFFFF:
        return 0
    return (mant * 2 ** (s % 256)) % 2**256


def test_compact_bits_every_exponent(ok, hs):
    for bits in _bits_cases():
        want = _python_compact(bits)
        assert oh.compact_target(bits) == want, hex(bits)
        for f in (ok.ok_pow_compact_target, hs.hs_compact_target):
            out = np.zeros(32, dtype=np.uint8)
            f(bits, out.ctypes.data)
            assert int.from_bytes(out.tobytes(), "little") == want, (f, hex(bits))


@pytest.mark.parametrize("fixture", oh.FIXTURES)
def test_fixture_header_hashes(ok, hs, fixture):
    _, hdrs = oh.fixture_headers(fixture)
    b = HeaderBatch.from_dicts(hdrs)
    par = b.parents if b.parents.size else np.zeros((1, 32), dtype=np.uint8)
    for i, h in enumerate(hdrs):
        rec = b.headers[i:i + 1]
        for f in (ok.ok_pow_header_hash, hs.hs_header_hash):
            out = np.zeros(32, dtype=np.uint8)
            f(rec.ctypes.data, par.ctypes.data, b.level_len.ctypes.data if b.level_len.size else None, h["nonce"], h["timestamp"], out.ctypes.data)
            assert out.tobytes() == h["hash"], (fixture, i)
        if i % 500 == 0:
            assert oh.block_hash(h) == h["hash"]


@pytest.mark.parametrize("fixture", oh.FIXTURES)
def test_fixture_headers_validate_alike(ok, hs, fixture):
    """Every header of a fixture through the C restatement; a sample through the host build and the Python restatement."""
    params, hdrs = oh.fixture_headers(fixture)
    b = HeaderBatch.from_dicts(hdrs)
    for skip in (False, True):
        rules = oh.fixture_rules(params, skip_pow=skip)
        res, hh, pw, pre = oh.oracle_validate(ok, b, rules)
        assert all(hh[i].tobytes() == h["hash"] for i, h in enumerate(hdrs))
        # the fixtures were made with skip_proof_of_work: their PoW does not meet their bits
        assert int(res["pow_passed"].sum()) == sum(1 for h in hdrs if not h["parents_by_level"])
        want_bad = 0 if skip else 6
        assert all(int(res["status"][i]) in (want_bad, 1) for i in range(len(hdrs)))
        for i in list(range(0, len(hdrs), max(1, len(hdrs) // 40)))[:40] + [len(hdrs) - 1]:
            r = np.zeros(1, dtype=HEADER_RESULT_DTYPE)
            p, q = np.zeros(32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
            par = b.parents if b.parents.size else np.zeros((1, 32), dtype=np.uint8)
            hs.hs_validate(b.headers[i:i + 1].ctypes.data, par.ctypes.data, b.level_len.ctypes.data if b.level_len.size else None,
                           ctypes.addressof(rules), r.ctypes.data, p.ctypes.data, q.ctypes.data)
            assert r.tobytes() == res[i:i + 1].tobytes() and p.tobytes() == pw[i].tobytes() and q.tobytes() == pre[i].tobytes(), (fixture, i)
        for i in (1, len(hdrs) // 2):
            rd = dict(block_version=1, max_block_parents=rules.max_block_parents, max_block_level=rules.max_block_level,
                      timestamp_deviation_tolerance=rules.timestamp_deviation_tolerance, now_ms=rules.now_ms, flags=rules.flags)
            pr = oh.check_pow(hdrs[i], rules.max_block_level)
            st = oh.validate_in_isolation(hdrs[i], rd, pr)
            assert (int(res["status"][i]), int(res["a"][i]), int(res["b"][i]), int(res["level"][i]), bool(res["pow_passed"][i])) == st
            assert int.from_bytes(pw[i].tobytes(), "little") == pr[1] and pre[i].tobytes() == pr[0]


def test_fixture_parent_levels_are_consistent(ok):
    """A block listed at parents_by_level[L] of a child is of level >= L (the reference builds level-L parents from blocks of level
    >= L): every fixture hash that appears at some L >= 1 has a computed level of at least L."""
    for fixture in oh.FIXTURES:
        params, hdrs = oh.fixture_headers(fixture)
        res, _, _, _ = oh.oracle_validate(ok, HeaderBatch.from_dicts(hdrs), oh.fixture_rules(params))
        level = {h["hash"]: int(res["level"][i]) for i, h in enumerate(hdrs)}
        seen = 0
        for h in hdrs:
            for L, ps in enumerate(h["parents_by_level"]):
                for p in ps if L >= 1 else ():
                    if p in level:
                        seen += 1
                        assert level[p] >= L, (fixture, p.hex(), L, level[p])
        assert seen > 100


def test_rules_in_order():
    """The Python restatement's rule order on mutated headers (the same cases run on the GPU in test_gpu_headers.py)."""
    _, hdrs = oh.fixture_headers(oh.FIXTURES[0])
    h = dict(hdrs[5])
    rd = dict(block_version=1, max_block_parents=len(h["parents_by_level"][0]), max_block_level=254, timestamp_deviation_tolerance=600,
              now_ms=h["timestamp"], flags=0)
    pr = (None, None, False, 3)
    assert oh.validate_in_isolation(h, rd, pr)[0] == oh.INVALID_POW
    assert oh.validate_in_isolation(h, dict(rd, flags=1), pr)[0] == oh.OK
    o = dict(h, parents_by_level=[h["parents_by_level"][0][:1] + [oh.ORIGIN]] + h["parents_by_level"][1:])
    assert oh.validate_in_isolation(o, rd, pr)[0] == oh.ORIGIN_PARENT
    assert oh.validate_in_isolation(h, dict(rd, max_block_parents=len(h["parents_by_level"][0]) - 1), pr)[:3] == (
        oh.TOO_MANY_PARENTS, len(h["parents_by_level"][0]), len(h["parents_by_level"][0]) - 1)
    assert oh.validate_in_isolation(dict(o, parents_by_level=[[]]), rd, pr)[0] == oh.NO_PARENTS
    t = dict(o, timestamp=h["timestamp"] + 600_001)
    assert oh.validate_in_isolation(t, rd, pr)[:3] == (oh.TIME_TOO_FAR_INTO_THE_FUTURE, t["timestamp"], h["timestamp"] + 600_000)
    assert oh.validate_in_isolation(dict(t, version=3), rd, pr)[:2] == (oh.WRONG_BLOCK_VERSION, 3)
