"""GPU-less unit tests of the comb key record and ladder (key_comb_build, ecmult_comb; DESIGN.md §4 K1): tests/hostsim/hostsim_comb.cpp
compiles the device headers with g++, generator entries are computed on demand, and every result is compared with pyref."""
import ctypes
import os
import random
import subprocess

import pytest

import pyref

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
P, N, G = pyref.P, pyref.N, pyref.G
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
KC_WORDS, KC_STATUS = 528, 512


@pytest.fixture(scope="module")
def comb():
    src, out = os.path.join(HS, "hostsim_comb.cpp"), os.path.join(HS, "libhostsim_comb.so")
    hdrs = [os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc", f) for f in ("kgv_arith.cuh", "kgv_secp.cuh", "kgv_sha256.cuh", "kgv_verify.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return ctypes.CDLL(out)


def words(x, n=8):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def num(w, lo, n=8):
    return sum(w[lo + i] << (32 * i) for i in range(n))


def record(lib, x, tag=2):
    be = (ctypes.c_uint32 * 8)(*[(x >> (32 * (7 - i))) & 0xFFFFFFFF for i in range(8)])
    rec = (ctypes.c_uint32 * KC_WORDS)()
    st = lib.hs_comb_build(be, tag, rec)
    return st, rec


def ecmult(lib, rec, kp, kg):
    xy = (ctypes.c_uint32 * 16)()
    inf = lib.hs_ecmult_comb(rec, words(kp), words(kg), xy)
    return None if inf else (num(xy, 0), num(xy, 8))


def expect(kp, pt, kg):
    return pyref.pt_add(pyref.pt_mul(kp % N, pt), pyref.pt_mul(kg % N, G))


def test_generator_table_bases(comb):
    for j in range(8):
        xy = (ctypes.c_uint32 * 16)()
        comb.hs_gtab_base(j, xy)
        assert (num(xy, 0), num(xy, 8)) == pyref.pt_mul(2 ** (32 * j), G)


def test_record_entries_are_true_affine(comb):
    rnd = random.Random(11)
    for tag in (2, 3):
        pt = pyref.pt_mul(rnd.randrange(1, N), G)
        st, rec = record(comb, pt[0], tag)
        assert st == 1
        y = pt[1] if (pt[1] & 1) == (tag == 3) else P - pt[1]
        base = (pt[0], y)
        for t in range(4):
            for e in range(8):
                x_, y_ = num(rec, 16 * (8 * t + e)), num(rec, 16 * (8 * t + e) + 8)
                assert (x_ % P, y_ % P) == pyref.pt_mul((2 * e + 1) << (32 * t), base), (t, e)


def test_record_bad_keys(comb):
    assert record(comb, P + 1)[0] == 2      # x >= p
    x = 5
    while pyref.lift_x(x) is not None:
        x += 1
    assert record(comb, x)[0] == 2          # not on the curve
    assert record(comb, G[0], 4)[0] == 2    # bad tag


def test_random_scalars(comb):
    rnd = random.Random(12)
    pt = pyref.pt_mul(rnd.randrange(1, N), G)
    st, rec = record(comb, pt[0], 2 + (pt[1] & 1))
    assert st == 1
    for _ in range(40):  # both parities of both GLV halves occur among these
        kp, kg = rnd.randrange(N), rnd.randrange(N)
        assert ecmult(comb, rec, kp, kg) == expect(kp, pt, kg)


def test_edge_scalars(comb):
    pt = pyref.pt_mul(0xC0FFEE, G)
    st, rec = record(comb, pt[0], 2 + (pt[1] & 1))
    top = 2 ** 128 - 1
    ks = [0, 1, 2, N - 1, N - 2, top, (top * LAMBDA) % N, (top + top * LAMBDA) % N, (top - top * LAMBDA) % N, 2 ** 255 % N]
    for kp in ks:
        for kg in (0, 1, N - 1, 2 ** 256 - 2 ** 128 - 1):
            assert ecmult(comb, rec, kp, kg % N) == expect(kp, pt, kg), (kp, kg)


def test_exact_special_cases(comb):
    # P = G, so the key and generator parts can meet
    st, rec = record(comb, G[0], 2)
    # kP = 2: m1 = 3 with the parity fix, k2 = 0: m2 = 1.  Before the fixes R = 3P + lambda*P + kG*G = -P: the first fix adds -P to -P (P + P)
    kg = (-(4 + LAMBDA)) % N
    assert ecmult(comb, rec, 2, kg) == expect(2, G, kg)
    # R = P - P at the last addition: the result is the point at infinity
    assert ecmult(comb, rec, 5, N - 5) is None
    assert ecmult(comb, rec, 0, 0) is None
    # kP = 0: the key part is P + lambda*P until the fixes; kG = -(1 + lambda) makes R infinite after the last generator addition, then
    # both fixes add onto the point at infinity
    kg = (-(1 + LAMBDA)) % N
    assert ecmult(comb, rec, 0, kg) == expect(0, G, kg)
