"""GPU-less unit tests of the joint table of comb records and its ladder (key_joint_build, recode_joint, ecmult_joint; DESIGN.md §4 K1):
tests/hostsim/hostsim_joint.cpp compiles the device headers with g++, generator entries are computed on demand, and every result is
compared with pyref, with the host build of ecmult_comb and with the scalar model of tests/joint_model.py."""
import ctypes
import os
import random
import subprocess

import pytest

import joint_model as jm
import ladder_model as lm
import pyref

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
P, N, G = pyref.P, pyref.N, pyref.G
LAMBDA = lm.LAMBDA
KJ_WORDS, KJ_JOINT, KC_STATUS = 2576, 528, 512
TOP = 2 ** 128 - 1
EDGE_KP = [0, 1, 2, N - 1, N - 2, TOP, (TOP * LAMBDA) % N, (TOP + TOP * LAMBDA) % N, (TOP - TOP * LAMBDA) % N, 2 ** 255 % N]
EDGE_KG = [0, 1, N - 1, (2 ** 256 - 2 ** 128 - 1) % N]


@pytest.fixture(scope="module")
def joint():
    src, out = os.path.join(HS, "hostsim_joint.cpp"), os.path.join(HS, "libhostsim_joint.so")
    hdrs = [os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc", f) for f in ("kgv_arith.cuh", "kgv_secp.cuh", "kgv_sha256.cuh", "kgv_verify.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    lib = ctypes.CDLL(out)
    assert lib.hs_kj_words() == KJ_WORDS
    return lib


def words(x, n=8):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def num(w, lo, n=8):
    return sum(w[lo + i] << (32 * i) for i in range(n))


def record(lib, x, tag=2):
    be = (ctypes.c_uint32 * 8)(*[(x >> (32 * (7 - i))) & 0xFFFFFFFF for i in range(8)])
    rec = (ctypes.c_uint32 * KJ_WORDS)()
    return lib.hs_joint_build(be, tag, rec), rec


def ecmult(lib, rec, kp, kg, which=0):
    xy = (ctypes.c_uint32 * 16)()
    inf = lib.hs_ecmult(rec, words(kp), words(kg), which, xy)
    return None if inf else (num(xy, 0), num(xy, 8))


def expect(kp, pt, kg):
    return pyref.pt_add(pyref.pt_mul(kp % N, pt), pyref.pt_mul(kg % N, G))


def key_point(seed):
    pt = pyref.pt_mul(seed, G)
    return pt, 2 + (pt[1] & 1)


def test_glv_halves_bound():
    # the bounds recode_joint's comment states: |k1| <= (a1 + a2)/2 + 1, |k2| <= (|b1| + b2)/2 + 1, both below 2^128
    assert (lm.A1 + lm.A2) // 2 + 1 < 2 ** 128 and (lm.MB1 + lm.A1) // 2 + 1 < 2 ** 128
    rnd = random.Random(31)
    for k in EDGE_KP + [rnd.randrange(N) for _ in range(2000)]:
        m1, _, m2, _ = lm.glv_split(k)
        assert m1 <= (lm.A1 + lm.A2) // 2 + 1 and m2 <= (lm.MB1 + lm.A1) // 2 + 1


def test_joint_entries(joint):
    rnd = random.Random(21)
    for tag in (2, 3):
        pt = pyref.pt_mul(rnd.randrange(1, N), G)
        st, rec = record(joint, pt[0], tag)
        assert st == 1
        y = pt[1] if (pt[1] & 1) == (tag == 3) else P - pt[1]
        for t in range(4):
            T = pyref.pt_mul(1 << (32 * t), (pt[0], y))
            for a in range(4):
                for k in range(8):
                    e = KJ_JOINT + 16 * (32 * t + 8 * a + k)
                    got = (num(rec, e) % P, num(rec, e + 8) % P)
                    assert got == pyref.pt_mul(((2 * a + 1) + (2 * k - 7) * LAMBDA) % N, T), (tag, t, a, k)


def test_bad_key_leaves_verdict(joint):
    assert record(joint, P + 1)[0] == 2
    assert record(joint, G[0], 4)[0] == 2


def _check_recoding(lib, m):
    h = (ctypes.c_uint32 * 5)()
    fix = lib.hs_recode_joint(words(m, 5), h)
    cs, mfix = jm.recode_joint(m)
    assert bool(fix) == mfix
    assert all(c % 2 == 1 and abs(c) < 2 ** 33 for c in cs)
    assert sum(c << (32 * t) for t, c in enumerate(cs)) == m + mfix
    assert num(h, 0, 5) == jm.packed(cs)
    # the digits round-trip: sum d * 2^(32t + 3w) = m (+1)
    assert sum(d << (32 * t + 3 * w) for t, c in enumerate(cs) for w, d in enumerate(jm.digits(c))) == m + mfix


def test_recoding_round_trips(joint):
    rnd = random.Random(22)
    ms = [0, 1, 2, 3, 2 ** 32 - 1, 2 ** 32, 2 ** 64, 2 ** 96 - 1, 2 ** 96, TOP, TOP - 1, (lm.A1 + lm.A2) // 2 + 1, (lm.MB1 + lm.A1) // 2 + 1]
    for k in EDGE_KP:
        m1, _, m2, _ = lm.glv_split(k)
        ms += [m1, m2]
    ms += [rnd.getrandbits(128) for _ in range(300)] + [rnd.getrandbits(rnd.randrange(1, 129)) for _ in range(300)]
    for m in ms:
        _check_recoding(joint, m)


def test_model_schedule_sums():
    rnd = random.Random(23)
    for _ in range(200):
        kp, kg, d = rnd.randrange(N), rnd.randrange(N), rnd.randrange(1, N)
        recs, _, final = lm.run(jm.ecmult_joint_ops(kp, kg), d)
        assert final == ((kp * d + kg) % N or None)
        assert sum(r["label"][0] == "key" for r in recs) == 44


def test_random_scalars(joint):
    rnd = random.Random(24)
    pt, tag = key_point(rnd.randrange(1, N))
    st, rec = record(joint, pt[0], tag)
    assert st == 1
    for _ in range(40):
        kp, kg = rnd.randrange(N), rnd.randrange(N)
        r = ecmult(joint, rec, kp, kg)
        assert r == expect(kp, pt, kg)
        assert r == ecmult(joint, rec, kp, kg, which=1)


def test_edge_scalars(joint):
    pt, tag = key_point(0xC0FFEE)
    st, rec = record(joint, pt[0], tag)
    for kp in EDGE_KP:
        for kg in EDGE_KG:
            r = ecmult(joint, rec, kp, kg)
            assert r == expect(kp, pt, kg), (kp, kg)
            assert r == ecmult(joint, rec, kp, kg, which=1)


def test_exact_special_cases(joint):
    # P = G: the key and generator parts can meet
    st, rec = record(joint, G[0], 2)
    for kp, kg in [(2, (-(4 + LAMBDA)) % N), (5, N - 5), (0, 0), (0, (-(1 + LAMBDA)) % N), (1, N - 1), (2, N - 2)]:
        assert ecmult(joint, rec, kp, kg) == expect(kp, G, kg), (kp, kg)
    # every exceptional addition the model finds on these and on the kP with both halves even (the combined parity fix), for P = G
    rnd = random.Random(25)
    cases = []
    for _ in range(50):
        kp = jm._u2_with_even_halves(rnd)
        ops = jm.ecmult_joint_ops(kp, 0)
        (a, b), (c, _) = lm.symbolic_before(ops, ("fix1", "fix2"))
        for sigma in (1, -1):
            cases.append((kp, (sigma * c - a) % N))  # d = 1: the accumulator before the fix is a + kG
        if len(cases) >= 8:
            break
    seen = set()
    for kp, kg in cases:
        recs, _, final = lm.run(jm.ecmult_joint_ops(kp, kg), 1)
        seen |= {e[2] for e in lm.events(recs)}
        assert ecmult(joint, rec, kp, kg) == expect(kp, G, kg), (kp, kg)
    assert {"dbl", "neg"} <= seen
