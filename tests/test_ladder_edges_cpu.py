"""GPU-less tests of the verify ladders' exceptional additions (doubling fall-through, cancellation to infinity, addition onto
infinity mid-ladder), on signatures built by tests/ladder_model.py to reach them.  The model itself is checked against the host build
of the device code (tests/hostsim) and against pyref points; then every crafted case goes through the host builds of both ladders,
the plain oracle, the oracle's fast port and pyref."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import ladder_model as L
import pyref

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
N, P, G = pyref.N, pyref.P, pyref.G
KC_WORDS = 528


def _build(name):
    src, out = os.path.join(HS, name + ".cpp"), os.path.join(HS, "lib" + name + ".so")
    hdrs = [os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc", f) for f in ("kgv_arith.cuh", "kgv_secp.cuh", "kgv_sha256.cuh", "kgv_verify.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def secp():
    return _build("hostsim_secp")


@pytest.fixture(scope="module")
def comb():
    return _build("hostsim_comb")


@pytest.fixture(scope="module")
def cases(oracle):
    return {"ecdsa": list(L.ecdsa_ladder_cases(oracle)) + L.ecdsa_edge_cases(),
            "schnorr": list(L.schnorr_ladder_cases(oracle)) + L.bip340_cases()}


def limbs(x, n=8):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def val(a):
    return sum(int(v) << (32 * i) for i, v in enumerate(a))


LAMBDA = L.LAMBDA
EDGE_SCALARS = [0, 1, 2, N - 1, N - 2, 2**128 - 1, 2**128, 2**128 + 1, LAMBDA, N - LAMBDA, (2**128 * LAMBDA) % N, (N - 1) // 2,
                (N + 1) // 2, 2**255 % N, (2**128 - 1) * (1 + LAMBDA) % N, (-(1 + LAMBDA)) % N, (-(4 + LAMBDA)) % N]


def test_model_product(oracle):
    """the final accumulator of both schedules is kP*d + kG, for random and edge scalars"""
    rnd = random.Random(21)
    pairs = [(a, b) for a in EDGE_SCALARS for b in (0, 1, N - 1, 2**256 - 2**128 - 1 - N, 0xFFFF0000FFFF)] + [(rnd.randrange(N), rnd.randrange(N)) for _ in range(300)]
    for kp, kg in pairs:
        d = rnd.randrange(1, N)
        for fn in L.SCHEDULES.values():
            recs, pre, fin = L.run(fn(kp, kg), d)
            assert fin == ((kp * d + kg) % N or None), (hex(kp), hex(kg))


def test_glv_split_matches_the_host_build(secp):
    rnd = random.Random(22)
    ks = EDGE_SCALARS + [rnd.randrange(N) for _ in range(3000)] + [rnd.randrange(2**128) for _ in range(200)]
    for k in ks:
        k1, k2 = (ctypes.c_uint32 * 5)(), (ctypes.c_uint32 * 5)()
        n1, n2 = ctypes.c_int(), ctypes.c_int()
        secp.hs_glv_split(limbs(k), k1, ctypes.byref(n1), k2, ctypes.byref(n2))
        assert (val(k1), bool(n1.value), val(k2), bool(n2.value)) == L.glv_split(k), hex(k)


def _host_trace(secp):
    def f(pk, msg, sig):
        out = (ctypes.c_uint32 * (32 * 16))()
        st = secp.hs_schnorr_trace(pk, msg, sig, out)
        return st, [list(out[16 * s:16 * s + 16]) for s in range(32)]
    return f


def test_schnorr_trace_matches_the_model(secp, oracle, cases):
    """hs_schnorr_trace (the host build of ecmult_double) against the model: split, flags, pre-fix accumulator"""
    from rusty_kaspa_b200 import workload as W
    trace = _host_trace(secp)
    crafted = [c for c in cases["schnorr"] if c["d"] is not None]
    for c in crafted:
        assert L.check_schnorr_trace(trace, c) == 0, c["label"]
    # ordinary signatures, with their discrete logs
    keys = W.ScalarPointPool(4, 23, b"keys")
    rnd = random.Random(23)
    for i in range(12):
        d, pk = keys.scalars[i % 4], keys.xs[i % 4]
        m = rnd.randbytes(32)
        sig = pyref.schnorr_sign(d.to_bytes(32, "big"), m)
        assert L.check_schnorr_trace(trace, {"pk": pk, "msg": m, "sig": sig, "d": d}) == 1


def _key_point(c):
    if c["kind"] == "ecdsa":
        return pyref.lift_x(int.from_bytes(c["pk"][1:], "big"), odd=c["pk"][0] == 3)
    return pyref.lift_x(int.from_bytes(c["pk"], "big"))


def _replay_points(c):
    """walks the case's schedule with pyref points (key multiples from the parsed key, generator multiples from G) and returns the
    exceptional additions seen: [(label, event)]"""
    Q = _key_point(c)
    kP, kG = (c["u2"], c["u1"]) if c["kind"] == "ecdsa" else (c["kP"], c["kG"])
    acc, seen, first = None, [], True
    for op in L.SCHEDULES[c["schedule"]](kP, kG):
        if op[0] == "dbl":
            for _ in range(op[1]):
                acc = pyref.pt_add(acc, acc)
            continue
        x = pyref.pt_add(pyref.pt_mul(op[2] % N, Q), pyref.pt_mul(op[3] % N, G))
        if acc is None and not first:
            seen.append((op[1], "inf"))
        elif acc is not None and acc == x:
            seen.append((op[1], "dbl"))
        elif acc is not None and acc[0] == x[0]:
            seen.append((op[1], "neg"))
        acc, first = pyref.pt_add(acc, x), False
    return seen


def test_claimed_coincidences_happen_on_the_curve(cases):
    """for a subset of the targeted cases, the coincidence the model claims happens between real points at the claimed addition"""
    targeted = [c for k in ("ecdsa", "schnorr") for c in cases[k] if c["target"] is not None and not c["label"].endswith("twin")]
    rnd = random.Random(24)
    for c in rnd.sample(targeted, 10) + [c for c in targeted if c["target"][0] == "fix2"][:2]:
        assert _replay_points(c) == [(lab, ev) for _, lab, ev in c["events"]], c["label"]


def _oracle_batches(oracle, kind, cases):
    pk, msg, sig = L.arrays(cases)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    out = []
    for fn in (f"ok_{kind}_verify_batch", f"ok_{kind}_verify_batch_fast"):
        st = np.zeros(len(cases), dtype=np.uint8)
        getattr(oracle, fn)(vp(pk), vp(msg), vp(sig), ctypes.c_size_t(len(cases)), vp(st), 4)
        out.append(st.tolist())
    return out


@pytest.mark.parametrize("kind", ["ecdsa", "schnorr"])
def test_crafted_verdicts(secp, oracle, cases, kind):
    """host build of the inline ladder (ecmult_double) == plain oracle == fast port == pyref == the constructed verdict"""
    cs = cases[kind]
    exp = [c["exp"] for c in cs]
    hs = secp.hs_ecdsa_verify if kind == "ecdsa" else secp.hs_schnorr_verify
    ref = pyref.ecdsa_verify if kind == "ecdsa" else pyref.schnorr_verify
    assert [hs(c["pk"], c["msg"], c["sig"]) for c in cs] == exp
    plain, fast = _oracle_batches(oracle, kind, cs)
    assert plain == exp and fast == exp
    assert [ref(c["pk"], c["msg"], c["sig"]) for c in cs] == exp


def test_comb_ladder_on_crafted_scalars(comb, cases):
    """the host build of ecmult_comb from the key's comb record, for every case with a known scalar pair, against pyref"""
    n = 0
    recs = {}
    for c in cases["ecdsa"] + cases["schnorr"]:
        if c["d"] is None:
            continue
        kP, kG = (c["u2"], c["u1"]) if c["kind"] == "ecdsa" else (c["kP"], c["kG"])
        key = c["pk"]
        if key not in recs:
            x = int.from_bytes(key[-32:], "big")
            be = (ctypes.c_uint32 * 8)(*[(x >> (32 * (7 - i))) & 0xFFFFFFFF for i in range(8)])
            rec = (ctypes.c_uint32 * KC_WORDS)()
            assert comb.hs_comb_build(be, key[0] if len(key) == 33 else 2, rec) == 1
            recs[key] = rec
        xy = (ctypes.c_uint32 * 16)()
        inf = comb.hs_ecmult_comb(recs[key], limbs(kP), limbs(kG), xy)
        got = None if inf else (val(xy[:8]), val(xy[8:]))
        assert got == pyref.pt_add(pyref.pt_mul(kP, _key_point(c)), pyref.pt_mul(kG, G)), c["label"]
        n += 1
    assert n > 250


def test_coverage(cases):
    """every targetable addition of each schedule has a case under each relation, and the ECDSA ones include valid signatures"""
    rnd = random.Random(25)
    u1 = L._u1_without_zero_digits(rnd)
    u2 = L._u2_with_even_halves(rnd)
    for sched, fn in L.SCHEDULES.items():
        want = {(lab, s) for lab in L.targetable(fn(u2, u1)) for s in (1, -1)}
        got = {(c["target"], c["sigma"]) for c in cases["ecdsa"] if c["schedule"] == sched}
        assert want <= got, sorted(want - got)[:5]
        assert len(want) == 2 * (74 if sched == "double" else 50)
        for c in cases["ecdsa"]:
            if c["schedule"] == sched and c["target"] is not None:
                assert (c["target"], "dbl" if c["sigma"] > 0 else "neg") in [(lab, ev) for _, lab, ev in c["events"]]
    valid = [c for c in cases["ecdsa"] if c["exp"] == 1 and c["target"] is not None]
    assert len(valid) >= 200
    labels = {c["label"] for c in cases["ecdsa"]}
    assert {"ecdsa R=inf", "ecdsa u1=0 m=0", "ecdsa u1=0 m=n", "ecdsa m>=n"} <= labels
    sch = {(c["schedule"], c["target"], c["sigma"]) for c in cases["schnorr"] if c["target"]}
    assert len(sch) == 16
    assert any(c["label"] == "schnorr R=inf" for c in cases["schnorr"])
    # skipped generator digits: a sparse u1 drops generator additions
    sparse = [c for c in cases["ecdsa"] if c["target"] and c["target"][0] in ("glo", "ghi", "gen")
              and sum(1 for k in range(16) if not (c["u1"] >> (16 * k)) & 0xFFFF) >= 4]
    assert len(sparse) >= 4
