"""Scalar model of the joint ladder (recode_joint, ecmult_joint in rusty_kaspa_b200/csrc/kgv_secp.cuh), in the op format of
ladder_model.py, and constructors of ECDSA signatures that reach its exceptional additions.

The joint ladder adds, at window w = 10..0 and per tooth t, one entry e0*T + e1*lambda*T (T = 2^(32t) P, e0, e1 the signed 3-bit digits
11t + w of the two GLV halves with their signs); three doublings between windows; the generator's fields at bits 32j+16.. between the
second and the third doubling before window 5, those at bits 32j.. after window 0; then at most one parity fix."""
import random

import ladder_model as lm
from ladder_model import LAMBDA, N, glv_split

M32 = (1 << 32) - 1


def recode_joint(m):
    """recode_joint: (c_0..c_3, fix) with m + fix = sum c_t 2^(32t), every c_t odd, |c_t| < 2^33"""
    fix = (m & 1) == 0
    r, cs = m + fix, []
    for _ in range(3):
        c, q = r & M32, r >> 32
        if q % 2 == 0:
            c, q = c - (1 << 32), q + 1
        cs.append(c)
        r = q
    cs.append(r)
    return cs, fix


def digits(c):
    """the 11 signed odd 3-bit digits of one tooth, low first"""
    v = (c + (1 << 33) - 1) // 2
    return [2 * ((v >> (3 * w)) & 7) - 7 for w in range(11)]


def packed(cs):
    """the 5 words recode_joint writes, as one integer (word q at bit 32q)"""
    h = 0
    for i in range(44):
        t, w = divmod(i, 11)
        v = (cs[t] + (1 << 33) - 1) // 2
        h |= ((v >> (3 * w)) & 7) << (32 * (i // 10) + 3 * (i % 10))
    return h


def ecmult_joint_ops(kP, kG):
    """ecmult_joint as ops: ("add", ("key", w, t), c, 0), ("add", ("gen", 5 or 0, j), 0, g), ("dbl", k), parity fix labels ("fix1",),
    ("fix2",) or ("fix1", "fix2") for the one combined addition"""
    m1, n1, m2, n2 = glv_split(kP)
    sg = (-1 if n1 else 1, -1 if n2 else 1)
    (c1, f1), (c2, f2) = recode_joint(m1), recode_joint(m2)
    dg = ([digits(c) for c in c1], [digits(c) for c in c2])
    ops = []

    def key(w):
        for t in range(4):
            ops.append(("add", ("key", w, t), (dg[0][t][w] * sg[0] + dg[1][t][w] * sg[1] * LAMBDA) << (32 * t), 0))

    def gen(sh, w):
        for j in range(8):
            dd = (kG >> (32 * j + sh)) & 0xFFFF
            if dd:
                ops.append(("add", ("gen", w, j), 0, dd << (32 * j)))

    key(10)
    for w in range(9, -1, -1):
        if w == 5:
            ops.append(("dbl", 2))
            gen(16, 5)
            ops.append(("dbl", 1))
        else:
            ops.append(("dbl", 3))
        key(w)
    gen(0, 0)
    if f1 and f2:
        ops.append(("add", ("fix1", "fix2"), -sg[0] - sg[1] * LAMBDA, 0))
    elif f1:
        ops.append(("add", ("fix1",), -sg[0], 0))
    elif f2:
        ops.append(("add", ("fix2",), -sg[1] * LAMBDA, 0))
    return ops


def _u2_with_even_halves(rnd):
    while True:
        u = rnd.randrange(1, N)
        m1, _, m2, _ = glv_split(u)
        if m1 % 2 == 0 and m2 % 2 == 0:
            return u


def ecdsa_targeted(cv, rnd, label, sigma):
    """a valid ECDSA signature and its invalid twin whose joint ladder meets relation sigma (+1: accumulator == addend, a doubling;
    -1: accumulator == -addend, infinity) at addition `label`, as ladder_model's cases"""
    fix_both = label == ("fix1", "fix2")
    for _ in range(200):
        u1 = lm._u1_without_zero_digits(rnd)
        u2 = _u2_with_even_halves(rnd) if fix_both else rnd.randrange(1, N)
        ops = ecmult_joint_ops(u2, u1)
        sb = lm.symbolic_before(ops, label)
        if sb is None or sb[0] is None:
            continue
        (a, b), (c, g) = sb
        if c:
            den = (a - sigma * c) % N
            if den == 0:
                continue
            d = -b * pow(den, -1, N) % N
        else:
            if a == 0:
                continue
            d = (sigma * g - b) * pow(a, -1, N) % N
        if d == 0:
            continue
        k = (u1 + u2 * d) % N
        r = int.from_bytes(cv.pub(k)[1:], "big") % N if k else rnd.randrange(1, N)
        if r == 0:
            continue
        s = r * pow(u2, -1, N) % N
        if s > N // 2:
            continue
        m = u1 * s % N
        recs, _, final = lm.run(ops, d)
        ev = lm.events(recs)
        tgt = [e for e in ev if e[1] == label]
        assert tgt and tgt[0][2] == ("dbl" if sigma > 0 else "neg"), (label, sigma, ev)
        pk = cv.pub(d)
        while True:
            f = rnd.randrange(2, N)
            if f * s % N <= N // 2 and f * r % N:
                break
        kw = dict(schedule="joint", target=label, sigma=sigma, events=ev, d=d, u1=u1, u2=u2)
        name = f"ecdsa joint {'/'.join(map(str, label))} {'dbl' if sigma > 0 else 'neg'}"
        if k == 0:
            assert final is None
            return [lm._case("ecdsa", pk, lm._b32(m), lm._b32(r) + lm._b32(s), 0, name, **kw)]
        return [lm._case("ecdsa", pk, lm._b32(m), lm._b32(r) + lm._b32(s), 1, name, **kw),
                lm._case("ecdsa", pk, lm._b32(f * m % N), lm._b32(f * r % N) + lm._b32(f * s % N), 0, name + " twin", **kw)]
    raise AssertionError(f"no ECDSA case for joint {label} {sigma}")


def ecdsa_joint_cases(oracle, seed=9):
    """the joint ladder's targetable additions: the first and last generator additions of both groups, a key addition of windows 4 and
    0, and the combined parity fix, each under both relations"""
    cv, rnd = lm._Curve(oracle), random.Random(seed)
    labels = [("gen", 5, 0), ("gen", 5, 7), ("key", 4, 2), ("key", 0, 3), ("gen", 0, 0), ("gen", 0, 7), ("fix1", "fix2")]
    out = []
    for label in labels:
        for sigma in (1, -1):
            out += ecdsa_targeted(cv, rnd, label, sigma)
    return out


def schnorr_infinity_and_fix_cases(oracle, seed=10):
    """Schnorr triples (all invalid) whose joint ladder ends in R = infinity (s = e*d), or meets the combined parity fix under both
    relations (s solved from the accumulator before it)"""
    cv, rnd = lm._Curve(oracle), random.Random(seed)
    out = []
    for _ in range(3):
        d, pk = lm._schnorr_key(cv, rnd)
        r32, m32 = lm._b32(rnd.randrange(1, lm.P)), lm._b32(rnd.getrandbits(256))
        e = lm._challenge(r32, pk, m32)
        out.append(lm._case("schnorr", pk, m32, r32 + lm._b32(e * d % N), 0, "schnorr joint R=inf", d=d))
    for sigma in (1, -1):
        while True:
            d, pk = lm._schnorr_key(cv, rnd)
            r32, m32 = lm._b32(rnd.randrange(1, lm.P)), lm._b32(rnd.getrandbits(256))
            e = lm._challenge(r32, pk, m32)
            m1, _, m2, _ = glv_split(-e % N)
            if m1 % 2 or m2 % 2:
                continue
            # before the fix the accumulator is a*d + s, the fix adds c*d: a + s/d = sigma*c
            (a, _), (c, _) = lm.symbolic_before(ecmult_joint_ops(-e % N, 0), ("fix1", "fix2"))
            s = (sigma * c - a) * d % N
            recs, _, _ = lm.run(ecmult_joint_ops(-e % N, s), d)
            ev = [x for x in lm.events(recs) if x[1] == ("fix1", "fix2")]
            if ev and ev[0][2] == ("dbl" if sigma > 0 else "neg"):
                out.append(lm._case("schnorr", pk, m32, r32 + lm._b32(s), 0, f"schnorr joint fix {'dbl' if sigma > 0 else 'neg'}", d=d))
                break
    return out
