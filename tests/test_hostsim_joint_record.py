"""GPU-less unit tests of the comb-form key record the device builds (key_joint_record_build, joint_table_build; DESIGN.md §4 K1):
tests/hostsim/hostsim_joint_record.cpp compiles the device headers with g++.  Every record is compared with one built by pyref (P, the
verdict, each of the 128 joint entries) and with the host-side reference pair (key_comb_build + key_joint_build); the joint ladder
reads it as the verify kernels do."""
import ctypes
import os
import random
import subprocess

import pytest

import pyref

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
P, N, G = pyref.P, pyref.N, pyref.G
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
BETA = 0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE
JR_WORDS, JR_P, JR_STATUS, JR_JOINT = 2080, 0, 16, 32
KJ_WORDS, KJ_JOINT = 2576, 528
TOP = 2 ** 128 - 1


@pytest.fixture(scope="module")
def jr():
    src, out = os.path.join(HS, "hostsim_joint_record.cpp"), os.path.join(HS, "libhostsim_joint_record.so")
    hdrs = [os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc", f) for f in ("kgv_arith.cuh", "kgv_secp.cuh", "kgv_sha256.cuh", "kgv_verify.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return ctypes.CDLL(out)


def words(x, n=8):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def num(w, lo, n=8):
    return sum(w[lo + i] << (32 * i) for i in range(n))


def be(x):
    return (ctypes.c_uint32 * 8)(*[(x >> (32 * (7 - i))) & 0xFFFFFFFF for i in range(8)])


def build(lib, x, tag):
    rec = (ctypes.c_uint32 * JR_WORDS)()
    return lib.hs_jr_build(be(x), tag, rec), rec


def ref_build(lib, x, tag):
    rec = (ctypes.c_uint32 * KJ_WORDS)()
    return lib.hs_ref_build(be(x), tag, rec), rec


def pyref_joint(pt):
    """the 128 joint entries of the key pt, entry 32t + 8a + k = (2a+1) T + (2k-7) lambda T, T = 2^(32t) pt: by additions only"""
    out = []
    T = pt
    for t in range(4):
        if t:
            for _ in range(32):
                T = pyref.pt_add(T, T)
        T2 = pyref.pt_add(T, T)
        odd = [T]
        for _ in range(3):
            odd.append(pyref.pt_add(odd[-1], T2))  # (2e+1) T, e = 0..3
        lam = [(BETA * x % P, y) for x, y in odd]  # (2e+1) lambda T
        for a in range(4):
            for k in range(8):
                b = 2 * k - 7
                B = lam[(abs(b) - 1) // 2]
                if b < 0:
                    B = (B[0], P - B[1])
                out.append(pyref.pt_add(odd[a], B))
    return out


def key_for(seed, tag):
    pt = pyref.pt_mul(seed, G)
    y = pt[1] if (pt[1] & 1) == (tag == 3) else P - pt[1]
    return (pt[0], y)


def test_layout_and_constants(jr):
    lay = (ctypes.c_uint32 * 6)()
    jr.hs_jr_layout(lay)
    assert list(lay) == [JR_WORDS, JR_P, JR_STATUS, JR_JOINT, KJ_WORDS, KJ_JOINT]
    assert (JR_JOINT * 4) % 64 == 0 and (JR_WORDS * 4) % 64 == 0  # 64-byte entries of 64-byte aligned records
    assert pyref.pt_mul(LAMBDA, G) == (BETA * G[0] % P, G[1])


def test_entries_by_formula(jr):
    # every joint entry of both tags against ((2a+1) + (2k-7) lambda) 2^(32t) P by scalar multiplication, P and the verdict in place
    rnd = random.Random(41)
    for tag in (2, 3):
        pt = key_for(rnd.randrange(1, N), tag)
        st, rec = build(jr, pt[0], tag)
        assert st == 1 and rec[JR_STATUS] == 1
        assert (num(rec, JR_P), num(rec, JR_P + 8)) == pt  # canonical, straight from the lift
        for t in range(4):
            T = pyref.pt_mul(1 << (32 * t), pt)
            for a in range(4):
                for k in range(8):
                    e = JR_JOINT + 16 * (32 * t + 8 * a + k)
                    got = (num(rec, e) % P, num(rec, e + 8) % P)
                    assert got == pyref.pt_mul(((2 * a + 1) + (2 * k - 7) * LAMBDA) % N, T), (tag, t, a, k)


def test_bad_keys_carry_verdict(jr):
    off = next(x for x in range(1, 100) if pyref.lift_x(x) is None)  # no point with this x
    for x, tag in [(P + 1, 2), (P, 3), (2 ** 256 - 1, 2), (off, 2), (off, 3), (G[0], 4), (G[0], 0), (G[0], 6)]:
        st, rec = build(jr, x, tag)
        assert st == 2 and rec[JR_STATUS] == 2, (x, tag)


def test_many_keys_against_pyref_and_reference(jr):
    # a few hundred random keys of both tags: every word of P and the verdict, every joint entry against pyref's record and against
    # the host-side reference pair's (the shared trick across teeth and the conversion to true affine together)
    rnd = random.Random(42)
    for i in range(300):
        tag = 2 + (i & 1)
        pt = key_for(rnd.randrange(1, N), tag)
        st, rec = build(jr, pt[0], tag)
        rst, ref = ref_build(jr, pt[0], tag)
        assert st == rst == 1
        assert [rec[JR_P + w] for w in range(16)] == [(pt[w // 8] >> (32 * (w % 8))) & 0xFFFFFFFF for w in range(16)]
        exp = pyref_joint(pt)
        for e in range(128):
            got = (num(rec, JR_JOINT + 16 * e) % P, num(rec, JR_JOINT + 16 * e + 8) % P)
            assert got == exp[e], (i, e)
            assert got == (num(ref, KJ_JOINT + 16 * e) % P, num(ref, KJ_JOINT + 16 * e + 8) % P), (i, e)


def test_ladder_reads_the_record(jr):
    # ecmult_joint from the record as ecmult_key calls it, against pyref: random scalars and the parity-fix cases (both halves even,
    # one even: joint entry resp. P from the record's head)
    rnd = random.Random(43)
    pt = key_for(rnd.randrange(1, N), 3)
    st, rec = build(jr, pt[0], 3)
    assert st == 1
    kps = [0, 1, 2, N - 1, N - 2, TOP, (TOP * LAMBDA) % N, (TOP + TOP * LAMBDA) % N, 2 ** 255 % N] + [rnd.randrange(N) for _ in range(24)]
    for kp in kps:
        kg = rnd.randrange(N)
        xy = (ctypes.c_uint32 * 16)()
        inf = jr.hs_jr_ecmult(rec, words(kp), words(kg), xy)
        exp = pyref.pt_add(pyref.pt_mul(kp, pt), pyref.pt_mul(kg, G))
        assert (None if inf else (num(xy, 0), num(xy, 8))) == exp, kp
