"""Scalar model of the verify ladders (ecmult_double, ecmult_comb in rusty_kaspa_b200/csrc/kgv_secp.cuh) and constructors of signatures
that reach their exceptional additions.

With the key's discrete log d known, every point of either ladder is a known multiple of G, so the whole ladder can be followed with
integers mod n: each addition is recorded with its label, the accumulator before it (a scalar, or None for the point at infinity) and
the addend's scalar.  The three exceptional cases of the mixed addition are then
  * "dbl": accumulator == addend (gej_add_ge falls through into a doubling),
  * "neg": accumulator == -addend (the result is the point at infinity),
  * "inf": an addition onto the point at infinity after the start of the ladder (after a "neg").
Random signatures reach each with probability about 2^-250; the constructors below solve for them instead.

ECDSA: u1 = m/s and u2 = r/s are both free, so any addition after the first generator addition can be targeted by solving the
collision for d, and the signature can still be made valid.
Schnorr: kP = -e with e a hash of (r, key, message), so only s is free, and a VALID signature would fix s = k + e*d: no valid
signature can be steered.  The reachable targets (all with an invalid verdict) are the last two generator additions, the two parity
fixes and R = infinity.

Pure Python (uses oracle/pyref.py and, for the fast point multiplications, the C oracle's ok_ecdsa_pubkey)."""
import ctypes
import functools
import hashlib
import random

import numpy as np

import pyref

N, P, G = pyref.N, pyref.P, pyref.G
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
BETA = 0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE
# KGV_G1_LIMBS, KGV_G2_LIMBS, KGV_A1_LIMBS, KGV_MB1_LIMBS, KGV_A2_LIMBS as integers
G1 = 0x3086D221A7D46BCDE86C90E49284EB153DAA8A1471E8CA7FE893209A45DBB031
G2 = 0xE4437ED6010E88286F547FA90ABFE4C4221208AC9DF506C61571B4AE8AC47F71
A1 = 0x3086D221A7D46BCDE86C90E49284EB15
MB1 = 0xE4437ED6010E88286F547FA90ABFE4C3
A2 = 0x114CA50F7A8E2F3F657C1108D9D44CFD8
M160 = (1 << 160) - 1


# ------------------------------------------------------------------------------------------------ scalar code, bit for bit
def glv_split(k):
    """glv_split: k (< 2^256) -> (|k1|, neg1, |k2|, neg2), with the 2^384 rounding and the 160-bit truncation of the device code"""
    t1, t2 = k * G1, k * G2
    c1 = (t1 >> 384) + ((t1 >> 383) & 1)
    c2 = (t2 >> 384) + ((t2 >> 383) & 1)
    k1 = (k - c1 * A1 - c2 * A2) & M160
    k2 = (c1 * MB1 - c2 * A1) & M160
    n1, n2 = k1 >> 159, k2 >> 159
    if n1:
        k1 = -k1 & M160
    if n2:
        k2 = -k2 & M160
    return k1, bool(n1), k2, bool(n2)


def recode_signed_odd(m):
    """recode_signed_odd: (h, fix)"""
    fix = (m & 1) == 0
    t = (m + fix) & M160
    return (t >> 1) | (1 << 131), fix


def recoded_digit(h, i):
    """recoded_digit: (table index 0..7, negative)"""
    v = (h >> (4 * i)) & 15
    neg = (v & 8) == 0
    return ((~v & 7) if neg else (v & 7)), neg


def _digit(h, i):
    idx, neg = recoded_digit(h, i)
    return -(2 * idx + 1) if neg else 2 * idx + 1


# ------------------------------------------------------------------------------------------------ the two addition schedules
# An op is ("dbl", k) for k doublings, or ("add", label, c, g): the addend is c*P + g*G (c, g integers), P = d*G the key.
def _halves(kP):
    m1, n1, m2, n2 = glv_split(kP)
    h1, f1 = recode_signed_odd(m1)
    h2, f2 = recode_signed_odd(m2)
    return (h1, h2), (-1 if n1 else 1, -1 if n2 else 1), (f1, f2)


def ecmult_double_ops(kP, kG):
    """ecmult_double: windows i = 32..0, four doublings between them; per window the k1 digit on P, the k2 digit on lambda*P, and
    when i % 4 == 0 and i < 32 the 16-bit generator digits dlo (table 0: G) and dhi (table 4: 2^128 G), zero digits skipped; then the
    parity fixes.  Runs in the inline and the plain-record forms."""
    h, sg, fix = _halves(kP)
    ops = []
    for i in range(32, -1, -1):
        if i != 32:
            ops.append(("dbl", 4))
        ops.append(("add", ("k1", i), _digit(h[0], i) * sg[0], 0))
        ops.append(("add", ("k2", i), _digit(h[1], i) * sg[1] * LAMBDA, 0))
        if i % 4 == 0 and i < 32:
            w16 = i >> 2
            dlo, dhi = (kG >> (16 * w16)) & 0xFFFF, (kG >> (128 + 16 * w16)) & 0xFFFF
            if dlo:
                ops.append(("add", ("glo", i), 0, dlo))
            if dhi:
                ops.append(("add", ("ghi", i), 0, dhi << 128))
    if fix[0]:
        ops.append(("add", ("fix1",), -sg[0], 0))
    if fix[1]:
        ops.append(("add", ("fix2",), -sg[1] * LAMBDA, 0))
    return ops


def ecmult_comb_ops(kP, kG):
    """ecmult_comb: window 8 adds the top digits (i = 32) of both halves from tooth 3; windows w = 7..0 (four doublings before each)
    add slots s = 0..7 (half s & 1, tooth t = s >> 1, digit 8t + w); at w = 4 and w = 0 the generator tables j = 0..7 follow with
    bits 32j+16.. resp. 32j.. of kG (zero digits skipped); then the parity fixes.  Runs in the comb form."""
    h, sg, fix = _halves(kP)
    lam = (1, LAMBDA)
    ops = [("add", ("key", 8, half), _digit(h[half], 32) * sg[half] * lam[half] << 96, 0) for half in (0, 1)]
    for w in range(7, -1, -1):
        ops.append(("dbl", 4))
        for s in range(8):
            half, t = s & 1, s >> 1
            ops.append(("add", ("key", w, s), _digit(h[half], 8 * t + w) * sg[half] * lam[half] << (32 * t), 0))
        if w % 4 == 0:
            for j in range(8):
                dd = (kG >> (32 * j + (16 if w else 0))) & 0xFFFF
                if dd:
                    ops.append(("add", ("gen", w, j), 0, dd << (32 * j)))
    for half in (0, 1):
        if fix[half]:
            ops.append(("add", ("fix1",) if half == 0 else ("fix2",), -sg[half] * lam[half], 0))
    return ops


SCHEDULES = {"double": ecmult_double_ops, "comb": ecmult_comb_ops}


def run(ops, d):
    """Follows the ladder for the key d*G.  Returns (records, prefix, final): records[j] = dict(pos, label, acc, addend, event) for the
    j-th addition, acc the accumulator before it (None = the point at infinity), event None, "dbl", "neg" or "inf"; prefix = the
    accumulator before the parity fixes, final = the result (None = infinity)."""
    acc, recs, prefix = None, [], None
    for op in ops:
        if op[0] == "dbl":
            if acc is not None:
                acc = acc * (1 << op[1]) % N
            continue
        label, c, g = op[1:]
        if label[0] in ("fix1", "fix2") and prefix is None:
            prefix = [acc]
        x = (c * d + g) % N
        before, ev = acc, None
        if acc is None:
            ev = "inf" if recs else None
            acc = x
        elif acc == x:
            ev, acc = "dbl", 2 * x % N
        elif acc == (N - x) % N:
            ev, acc = "neg", None
        else:
            acc = (acc + x) % N
        recs.append({"pos": len(recs), "label": label, "acc": before, "addend": x, "event": ev})
    return recs, (prefix[0] if prefix else acc), acc


def events(recs):
    """the exceptional additions of a run: [(pos, label, event)]"""
    return [(r["pos"], r["label"], r["event"]) for r in recs if r["event"]]


def symbolic_before(ops, label):
    """Accumulator before the addition `label` as (a, b) with value a*d + b, assuming no exceptional addition before it (the generic
    case), plus the addend as (c, g).  None if the accumulator is the point at infinity there or the label is not in the schedule."""
    acc = None
    for op in ops:
        if op[0] == "dbl":
            if acc is not None:
                acc = (acc[0] << op[1], acc[1] << op[1])
            continue
        if op[1] == label:
            return (None if acc is None else (acc[0] % N, acc[1] % N)), (op[2] % N, op[3] % N)
        acc = (op[2], op[3]) if acc is None else (acc[0] + op[2], acc[1] + op[3])
    return None


def targetable(ops):
    """labels of the additions from the first generator addition on (the ones a choice of d can steer)"""
    out, seen = [], False
    for op in ops:
        if op[0] == "add":
            seen = seen or op[3] != 0
            if seen:
                out.append(op[1])
    return out


# ------------------------------------------------------------------------------------------------ helpers
def _b32(x):
    return x.to_bytes(32, "big")


class _Curve:
    """x and y parity of k*G through the C oracle (fast), pyref as the fall-back of nothing: the oracle is required"""

    def __init__(self, oracle):
        self.o = oracle

    def pub(self, k):
        """33-byte compressed k*G (k in [1, n))"""
        out = ctypes.create_string_buffer(33)
        assert self.o.ok_ecdsa_pubkey(_b32(k), out) == 1
        return out.raw


def _challenge(r32, pk32, m32):
    return int.from_bytes(pyref.tagged_hash("BIP0340/challenge", r32 + pk32 + m32), "big") % N


def _field(x, pos):
    return (x >> pos) & 0xFFFF


def _u1_without_zero_digits(rnd):
    while True:
        u = rnd.randrange(1, N)
        if all(_field(u, 16 * k) for k in range(16)):
            return u


def _u2_with_even_halves(rnd):
    while True:
        u = rnd.randrange(1, N)
        _, _, fix = _halves(u)
        if fix[0] and fix[1]:
            return u


def _case(kind, pk, msg, sig, exp, label, **kw):
    c = {"kind": kind, "pk": pk, "msg": msg, "sig": sig, "exp": exp, "label": label, "schedule": None, "target": None, "sigma": 0,
         "events": [], "d": None}
    c.update(kw)
    return c


# ------------------------------------------------------------------------------------------------ ECDSA
def _ecdsa_targeted(cv, rnd, sched, label, sigma, u1_fn):
    """a valid signature and its invalid twin whose `sched` ladder meets relation sigma at addition `label`"""
    ops_fn = SCHEDULES[sched]
    fix_target = label[0] in ("fix1", "fix2")
    for _ in range(200):
        u1 = u1_fn(rnd)
        u2 = _u2_with_even_halves(rnd) if fix_target else rnd.randrange(1, N)
        ops = ops_fn(u2, u1)
        sb = symbolic_before(ops, label)
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
        # k = 0 when the target is the last addition under sigma = -1: R is the point at infinity, no signature can be valid
        k = (u1 + u2 * d) % N
        r = int.from_bytes(cv.pub(k)[1:], "big") % N if k else rnd.randrange(1, N)
        if r == 0:
            continue
        s = r * pow(u2, -1, N) % N
        if s > N // 2:
            continue
        m = u1 * s % N
        recs, _, final = run(ops, d)
        ev = events(recs)
        tgt = [e for e in ev if e[1] == label]
        assert tgt and tgt[0][2] == ("dbl" if sigma > 0 else "neg"), (sched, label, sigma, ev)
        pk = cv.pub(d)
        while True:  # the twin: (f*r, f*s, f*m) has the same u1, u2 and a wrong r
            f = rnd.randrange(2, N)
            if f * s % N <= N // 2 and f * r % N:
                break
        kw = dict(schedule=sched, target=label, sigma=sigma, events=ev, d=d, u1=u1, u2=u2)
        name = f"ecdsa {sched} {'/'.join(map(str, label))} {'dbl' if sigma > 0 else 'neg'}"
        if k == 0:
            assert final is None
            return [_case("ecdsa", pk, _b32(m), _b32(r) + _b32(s), 0, name, **kw)]
        return [_case("ecdsa", pk, _b32(m), _b32(r) + _b32(s), 1, name, **kw),
                _case("ecdsa", pk, _b32(f * m % N), _b32(f * r % N) + _b32(f * s % N), 0, name + " twin", **kw)]
    raise AssertionError(f"no ECDSA case for {sched} {label} {sigma}")


def _ecdsa_signed(cv, rnd, d, m_red, msg_int, label):
    """a standard signature of message m_red (reduced) by key d, given as the 32-byte integer msg_int, and an invalid twin"""
    while True:
        k = rnd.randrange(1, N)
        r = int.from_bytes(cv.pub(k)[1:], "big") % N
        if r == 0:
            continue
        s = pow(k, -1, N) * (m_red + r * d) % N
        if s == 0:
            continue
        s = min(s, N - s)
        break
    pk = cv.pub(d)
    u1, u2 = m_red * pow(s, -1, N) % N, r * pow(s, -1, N) % N
    evs = {sched: events(run(fn(u2, u1), d)[0]) for sched, fn in SCHEDULES.items()}
    kw = dict(d=d, u1=u1, u2=u2, events=evs)
    return [_case("ecdsa", pk, _b32(msg_int), _b32(r) + _b32(s), 1, label, **kw),
            _case("ecdsa", pk, _b32(msg_int), _b32((r + 1) % N or 1) + _b32(s), 0, label + " twin", **kw)]


@functools.lru_cache(maxsize=None)
def _ecdsa_cases_cached(oracle_id, seed):
    return _build_ecdsa_cases(_ORACLES[oracle_id], seed)


_ORACLES = {}


def ecdsa_ladder_cases(oracle, seed=5):
    """Every targetable addition of both schedules under both relations (a valid signature and its invalid twin each), the final
    R = infinity, u1 = 0 (m = 0 and m = n), m >= n and u1 with zero 16-bit digits.  Cached per process."""
    _ORACLES[id(oracle)] = oracle
    return _ecdsa_cases_cached(id(oracle), seed)


def _build_ecdsa_cases(oracle, seed):
    cv, rnd = _Curve(oracle), random.Random(seed)
    out = []
    for sched, fn in SCHEDULES.items():
        # the labels are the same for every u1 without zero digits and every u2 with even halves
        labels = targetable(fn(_u2_with_even_halves(rnd), _u1_without_zero_digits(rnd)))
        for label in labels:
            for sigma in (1, -1):
                out += _ecdsa_targeted(cv, rnd, sched, label, sigma, _u1_without_zero_digits)

        # u1 with zero 16-bit digits: those generator additions are skipped; target the addition after a skipped one
        def sparse_u1(r):
            u = _u1_without_zero_digits(r)
            for k in r.sample(range(16), 6):
                u &= ~(0xFFFF << (16 * k))
            return u or 1
        for sigma in (1, -1):
            u1 = sparse_u1(rnd)
            lab = [l for l in targetable(fn(1, u1)) if l[0] in ("glo", "ghi", "gen")]
            out += _ecdsa_targeted(cv, rnd, sched, rnd.choice(lab[1:] or lab), sigma, lambda r, u=u1: u)
    # the final R = infinity: u1 = -u2*d
    for _ in range(4):
        d, r, s = rnd.randrange(1, N), rnd.randrange(1, N), rnd.randrange(1, N // 2)
        m = -r * d % N
        u1, u2 = m * pow(s, -1, N) % N, r * pow(s, -1, N) % N
        assert (u1 + u2 * d) % N == 0
        evs = {sc: events(run(fn(u2, u1), d)[0]) for sc, fn in SCHEDULES.items()}
        out.append(_case("ecdsa", cv.pub(d), _b32(m), _b32(r) + _b32(s), 0, "ecdsa R=inf", d=d, u1=u1, u2=u2, events=evs))
    # u1 = 0 (no generator additions), through m = 0 and m = n
    for msg_int in (0, N):
        for _ in range(2):
            out += _ecdsa_signed(cv, rnd, rnd.randrange(1, N), 0, msg_int, f"ecdsa u1=0 m={'0' if msg_int == 0 else 'n'}")
    # m >= n: the message reduces
    for _ in range(4):
        m_red = rnd.randrange(0, 2**256 - N)
        out += _ecdsa_signed(cv, rnd, rnd.randrange(1, N), m_red, m_red + N, "ecdsa m>=n")
    return tuple(out)


def crafted_ecdsa_edge_cases():
    """Triples built for the branches random data never reaches (big-integer arithmetic of oracle/pyref.py, no GPU / C code involved):
      * x(R) >= n, so that r = x(R) - n and the verifier must try r + n < p  (Q is SOLVED for: Q = r^-1 (s R - m G), no discrete log needed)
      * s exactly (n-1)/2 (the largest low S: valid) and (n+1)/2 (the smallest high S: rejected although the equation holds)
      * 33-byte keys with the uncompressed / hybrid tags 04, 06, 07 (PublicKey::from_slice fails on a 33-byte slice with those tags)
    Returns [(pk33, msg32, sig64, expected status, label)]."""
    rng = np.random.default_rng(77)
    out = []
    comp = lambda pt: bytes([2 + (pt[1] & 1)]) + pt[0].to_bytes(32, "big")
    j = 0
    while len([o for o in out if o[4] == "wrap"]) < 12:
        j += 1
        R = pyref.lift_x(N + int(rng.integers(1, 2**62)) * 7 + j)
        if R is None:
            continue
        r = R[0] - N
        s = int.from_bytes(rng.bytes(32), "big") % (N // 2 - 1) + 1  # low S
        m = int.from_bytes(rng.bytes(32), "big") % N
        Q = pyref.pt_mul(pow(r, -1, N), pyref.pt_add(pyref.pt_mul(s, R), pyref.pt_mul((N - m) % N, G)))
        sig = r.to_bytes(32, "big") + s.to_bytes(32, "big")
        out.append((comp(Q), m.to_bytes(32, "big"), sig, 1, "wrap"))
        out.append((comp(Q), ((m + 1) % N).to_bytes(32, "big"), sig, 0, "wrap-wrong-msg"))
    for target, exp in (((N - 1) // 2, 1), ((N + 1) // 2, 0), ((N - 1) // 2 - 1, 1), ((N + 1) // 2 + 1, 0)):
        for _ in range(6):
            d, k = int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1, int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1
            r = pyref.pt_mul(k, G)[0] % N
            m = (target * k - r * d) % N  # s = k^-1 (m + r d) = target
            out.append((comp(pyref.pt_mul(d, G)), m.to_bytes(32, "big"), r.to_bytes(32, "big") + target.to_bytes(32, "big"), exp, f"s={'low' if exp else 'high'}-boundary"))
    base = out[0]
    for tag in (0x04, 0x06, 0x07, 0x00, 0x05):
        out.append((bytes([tag]) + base[0][1:], base[1], base[2], 2, f"tag {tag:02x}"))
    return out


# ------------------------------------------------------------------------------------------------ Schnorr
def _schnorr_key(cv, rnd):
    d0 = rnd.randrange(1, N)
    pk = cv.pub(d0)
    return (N - d0 if pk[0] == 3 else d0), pk[1:]


def _schnorr_solve_s(sched, label, sigma, d, e):
    """s such that the `sched` ladder of R = s*G - e*P meets relation sigma at `label`, or None when this e admits none.
    Before the last two generator additions (no doublings after them) the accumulator is a*d + (s without their 16-bit fields); before
    a parity fix it is a*d + s."""
    kP = -e % N
    _, sg, fix = _halves(kP)
    if label[0] in ("fix1", "fix2"):
        if not (fix[0] and fix[1]):
            return None
        a, (c, _) = symbolic_before(SCHEDULES[sched](kP, 0), label)
        return (sigma * c - a[0]) * d % N
    p_last, p_prev = (128, 0) if sched == "double" else (224, 192)
    # all key digits are in before the last generator additions: -e, plus what the fixes take off again
    X = -(-e + sg[0] * fix[0] + sg[1] * LAMBDA * fix[1]) * d % N
    if label in (("ghi", 0), ("gen", 0, 7)):
        # s - g*2^p_last = sigma*g*2^p_last - a*d: the field g of s is solved directly
        g = (-sigma * _field(X, p_last)) & 0xFFFF
        s = (X + ((1 + sigma) * g << p_last)) % N
        return s if g and _field(s, p_last) == g else None
    # the one before the last: s without both fields = sigma*g*2^p_prev - a*d must have both fields zero, which fixes g and leaves
    # a 16-bit condition on e (about one e in 65 536); the last field is free
    g = (-sigma * _field(X, p_prev)) & 0xFFFF
    Y = (X + sigma * (g << p_prev)) % N
    if not g or _field(Y, p_prev) or _field(Y, p_last):
        return None
    s = Y + (g << p_prev) + (0x5A5A << p_last)
    return s if s < N else None


def _schnorr_targeted(cv, rnd, sched, label, sigma):
    for _ in range(20):
        d, pk = _schnorr_key(cv, rnd)
        r32 = _b32(rnd.randrange(1, P))
        pre = hashlib.sha256(hashlib.sha256(b"BIP0340/challenge").digest() * 2)
        pre.update(r32 + pk)
        for _ in range(1 << 20):
            m32 = _b32(rnd.getrandbits(256))
            h = pre.copy()
            h.update(m32)
            e = int.from_bytes(h.digest(), "big") % N
            s = _schnorr_solve_s(sched, label, sigma, d, e)
            if s is not None:
                break
        else:
            continue
        assert e == _challenge(r32, pk, m32)
        recs, _, final = run(SCHEDULES[sched](-e % N, s), d)
        ev = events(recs)
        tgt = [x for x in ev if x[1] == label]
        if not tgt or tgt[0][2] != ("dbl" if sigma > 0 else "neg"):
            continue
        name = f"schnorr {sched} {'/'.join(map(str, label))} {'dbl' if sigma > 0 else 'neg'}"
        return _case("schnorr", pk, m32, r32 + _b32(s), 0, name, schedule=sched, target=label, sigma=sigma, events=ev, d=d, kP=-e % N, kG=s)
    raise AssertionError(f"no Schnorr case for {sched} {label} {sigma}")


@functools.lru_cache(maxsize=None)
def _schnorr_cases_cached(oracle_id, seed):
    oracle = _ORACLES[oracle_id]
    cv, rnd = _Curve(oracle), random.Random(seed)
    out = []
    for sched in SCHEDULES:
        last = [("glo", 0), ("ghi", 0)] if sched == "double" else [("gen", 0, 6), ("gen", 0, 7)]
        for label in last + [("fix1",), ("fix2",)]:
            for sigma in (1, -1):
                out.append(_schnorr_targeted(cv, rnd, sched, label, sigma))
    for _ in range(3):  # R = infinity: s = e*d
        d, pk = _schnorr_key(cv, rnd)
        r32, m32 = _b32(rnd.randrange(1, P)), _b32(rnd.getrandbits(256))
        e = _challenge(r32, pk, m32)
        s = e * d % N
        evs = {sc: events(run(fn(-e % N, s), d)[0]) for sc, fn in SCHEDULES.items()}
        out.append(_case("schnorr", pk, m32, r32 + _b32(s), 0, "schnorr R=inf", d=d, kP=-e % N, kG=s, events=evs))
    return tuple(out)


def schnorr_ladder_cases(oracle, seed=6):
    """The last two generator additions, both parity fixes (each under both relations) of both schedules, and R = infinity: all
    invalid.  Cached per process."""
    _ORACLES[id(oracle)] = oracle
    return _schnorr_cases_cached(id(oracle), seed)


def bip340_cases():
    """rows 0-14 of BIP-340's test vectors, as cases"""
    from golden_util import bip340_vectors
    pk, msg, sig, exp, comments = bip340_vectors()
    return [_case("schnorr", pk[i].tobytes(), msg[i].tobytes(), sig[i].tobytes(), exp[i], f"bip340 row {i}: {comments[i]}") for i in range(len(exp))]


def ecdsa_edge_cases():
    """crafted_ecdsa_edge_cases as cases"""
    return [_case("ecdsa", k, m, s, e, "edge " + l) for (k, m, s, e, l) in crafted_ecdsa_edge_cases()]


def _val(words):
    return sum(int(v) << (32 * i) for i, v in enumerate(words))


def _prefix_point(tr):
    """the pre-fix accumulator of a trace (stages 15-17 on the isomorphic curve, true Z = Z * zs with zs at stage 13)"""
    X, Y, Z, zs = (_val(tr[s][:8]) for s in (15, 16, 17, 13))
    z = Z * zs % P
    if z == 0:
        return None
    zi = pow(z, -1, P)
    return (X * zi * zi % P, Y * zi * zi * zi % P)


def check_schnorr_trace(trace_fn, c):
    """trace_fn(pk, msg, sig) -> (status, trace[32][16]) as kgv_debug_schnorr_trace / hs_schnorr_trace give it, for a Schnorr case
    with a known key d: asserts that the GLV halves (stages 10, 11), the flags neg1, neg2, fix1, fix2 (stage 12) and the accumulator
    before the parity fixes (stages 15-17) are the model's.  Returns the status."""
    st, tr = trace_fn(c["pk"], c["msg"], c["sig"])
    d = c["d"]
    e = _challenge(c["sig"][:32], c["pk"], c["msg"])
    kP, kG = -e % N, int.from_bytes(c["sig"][32:], "big")
    m1, n1, m2, n2 = glv_split(kP)
    _, f1 = recode_signed_odd(m1)
    _, f2 = recode_signed_odd(m2)
    assert [int(v) for v in tr[12][:4]] == [n1, n2, f1, f2]
    assert _val(tr[10][:5]) == m1 and _val(tr[11][:5]) == m2
    _, pre, fin = run(ecmult_double_ops(kP, kG), d)
    if pre is not None:
        assert _prefix_point(tr) == pyref.pt_mul(pre, G)
    return st


def arrays(cases):
    """(pk, msg, sig) uint8 arrays of a list of cases of one kind"""
    klen = 33 if cases[0]["kind"] == "ecdsa" else 32
    f = lambda key, w: np.frombuffer(b"".join(c[key] for c in cases), dtype=np.uint8).reshape(-1, w).copy()
    return f("pk", klen), f("msg", 32), f("sig", 64)
