"""GPU-less unit tests of the device group law (gej_double_n, gej_add_ge) and of the one-fold wide accumulator
(fe_fold) it is built from: tests/hostsim/hostsim_group.cpp compiles the CUDA headers with g++ using the portable
primitive bodies, and every result is checked against Python integers and pyref's affine group law, including the
exact special cases (infinity, P + P, P - P) and non-canonical (weakly reduced) inputs."""
import ctypes
import os
import random
import subprocess

import pytest

import pyref

P = pyref.P
HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")


@pytest.fixture(scope="module")
def grp(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostsim") / "libhostsim_group.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HS, "hostsim_group.cpp")], check=True)
    return ctypes.CDLL(out)


def le(x):
    return x.to_bytes(32, "little")


def weak(rnd, x):
    """x mod p as any representative in [0, 2^256)"""
    x %= P
    return x + P if x < 2**256 - P and rnd.random() < 0.3 else x


def to_gej(rnd, pt):
    if pt is None:
        return bytearray(96) + b"\x01"
    z = rnd.choice([1, rnd.randrange(1, P), P - 1])
    x, y = pt[0] * z * z % P, pt[1] * z * z * z % P
    return bytearray(le(weak(rnd, x)) + le(weak(rnd, y)) + le(weak(rnd, z)) + b"\x00")


def from_gej(b):
    if b[96]:
        return None
    x, y, z = (int.from_bytes(bytes(b[32 * i:32 * i + 32]), "little") for i in range(3))
    zi = pow(z, -1, P)
    return (x * zi * zi % P, y * zi * zi * zi % P)


def rand_point(rnd):
    return pyref.pt_mul(rnd.randrange(1, pyref.N), pyref.G)


def test_fold_wide_accumulator(grp):
    rnd = random.Random(11)
    lows = [0, 1, 2**32 + 976, 2**256 - 1, P, P - 1, 2**256 - 2**40, (2**160 - 1) << 96, 2**96 - 1]
    cases = [(v, t) for v in lows for t in range(-8, 9)]
    cases += [(rnd.randrange(2**256), rnd.randrange(-8, 9)) for _ in range(3000)]
    # carry (+1) / borrow (-1) out of limb 2, propagating into limbs 3..7 and sometimes past 2^256
    cases += [((2**96 - rnd.randrange(1, 2**36)) | (rnd.choice([rnd.randrange(2**160), 2**160 - 1]) << 96), rnd.randrange(1, 9)) for _ in range(300)]
    cases += [(rnd.randrange(2**36) | (rnd.choice([rnd.randrange(2**160), 0, 1 << 64]) << 96), rnd.randrange(-8, 0)) for _ in range(300)]
    o = ctypes.create_string_buffer(32)
    for v, t in cases:
        grp.hs_fe_fold(le(v), ctypes.c_int32(t), o)
        r = int.from_bytes(o.raw, "little")
        assert r < 2**256 and r % P == (v + t * 2**256) % P, (hex(v), t)


def test_doubling(grp):
    rnd = random.Random(12)
    for _ in range(60):
        pt, n = rand_point(rnd), rnd.choice([1, 2, 4])
        b = to_gej(rnd, pt)
        buf = ctypes.create_string_buffer(bytes(b), 97)
        grp.hs_gej_double_n(buf, n)
        exp = pyref.pt_mul(2**n, pt)
        assert from_gej(buf.raw) == exp
    buf = ctypes.create_string_buffer(bytes(to_gej(rnd, None)), 97)
    grp.hs_gej_double_n(buf, 4)
    assert buf.raw[96] == 1


def test_mixed_addition_and_its_special_cases(grp):
    rnd = random.Random(13)
    h = ctypes.create_string_buffer(32)
    for k in range(80):
        addend = rand_point(rnd)
        # r (Jacobian) += addend (affine): P + P, P - P, inf + Q, then P + Q
        r = {0: addend, 1: (addend[0], P - addend[1]), 2: None}.get(k % 8) if k % 8 < 3 else rand_point(rnd)
        buf = ctypes.create_string_buffer(bytes(to_gej(rnd, r)), 97)
        z1 = int.from_bytes(buf.raw[64:96], "little")
        grp.hs_gej_add_ge(buf, le(weak(rnd, addend[0])), le(weak(rnd, addend[1])), h)
        assert from_gej(buf.raw) == pyref.pt_add(r, addend), k
        if r is not None and from_gej(buf.raw) is not None:   # Z3 = Z1 * H
            z3 = int.from_bytes(buf.raw[64:96], "little")
            assert z3 % P == z1 * int.from_bytes(h.raw, "little") % P, k
