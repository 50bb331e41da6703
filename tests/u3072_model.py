"""Bit-exact model of the MuHash field product (u3072_mul_mod and u3072_coop_mul_mod, rusty_kaspa_b200/csrc/kgv_u3072.cuh).

Both multipliers fold the 6144-bit product with 2^3072 == PRIME_DIFF (mod p) until it is below 2^3072, and never reduce below p,
so each must return exactly `fold(a * b)`.  Their rare paths are a third fold round, a block carry rippling into an all-ones limb
block (the cooperative phases 2b and 3b), and the per-thread fold's second-round addition carrying out of limb block 0.  Random
(hashed) operands reach them with probability around 2^-3000, so `edge_cases` builds operands that do, and `paths` says which
paths a pair takes.  The tests compare the host build and the device kernels with `fold` exactly.
"""
import random

PRIME_DIFF = 1103717
P = 2**3072 - PRIME_DIFF
TOP = 2**3072
ONES = TOP - 1
B256 = 2**256


def fold(v):
    """v folded with 2^3072 == PRIME_DIFF until below 2^3072 (congruent to v mod p, not necessarily below p)."""
    while v >= TOP:
        v = (v % TOP) + (v >> 3072) * PRIME_DIFF
    return v


def _blocks(x, n):
    return [(x >> (256 * i)) % B256 for i in range(n)]


def _ripple(w, carry):
    """phase 2b / 3b: block carries rippled upwards; returns (final carry, whether an added carry left its block)."""
    cin, spilled = 0, False
    for k in range(len(w)):
        ov = 0
        if cin:
            s = w[k] + cin
            w[k], ov = s % B256, s >> 256
            spilled |= bool(ov)
        cin = carry[k] + ov
    return cin, spilled


def paths(a, b):
    """The rare paths the pair (a, b) takes in the two multipliers (both operands below 2^3072):
    'rounds'  fold rounds until below 2^3072 (2 is the common case; 3 runs `while (carry)` / `while (f)` twice),
    'ripple2b' a phase-2b block carry left the block it was added to (added into an all-ones block),
    'ripple3b' the same in phase 3b,
    'past0'   a second-round addition of the per-thread fold carried out of limb block 0."""
    assert 0 <= a < TOP and 0 <= b < TOP
    A, B = _blocks(a, 12), _blocks(b, 12)
    cols = [sum(A[i] * B[k - i] for i in range(max(0, k - 11), min(k, 11) + 1)) for k in range(23)]
    w, carry = [], []
    for k in range(24):  # phase 2: block k from the three column pieces that overlap it
        x = (cols[k] % B256 if k <= 22 else 0) + ((cols[k - 1] >> 256) % B256 if k >= 1 else 0) + (cols[k - 2] >> 512 if k >= 2 else 0)
        w.append(x % B256)
        carry.append(x >> 256)
    out, r2b = _ripple(w, carry)
    assert out == 0 and sum(v << (256 * k) for k, v in enumerate(w)) == a * b
    w3, carry3 = [], []
    for k in range(12):  # phase 3: fold block 12 + k into block k
        x = w[k] + w[12 + k] * PRIME_DIFF
        w3.append(x % B256)
        carry3.append(x >> 256)
    f, r3b = _ripple(w3, carry3)
    v = sum(x << (256 * k) for k, x in enumerate(w3))
    assert f == (a * b % TOP + (a * b >> 3072) * PRIME_DIFF) >> 3072
    rounds, past0 = 1, False
    while f:  # the second-round addition, limb block by limb block, exactly as u3072_fold's `while (carry)`
        rounds += 1
        s = v % B256 + f * PRIME_DIFF
        past0 |= s >= B256
        v = v + f * PRIME_DIFF
        f, v = v >> 3072, v % TOP
    assert v == fold(a * b)
    return {"rounds": rounds, "ripple2b": r2b, "ripple3b": r3b, "past0": past0}


FLAGS = {"round3": lambda p: p["rounds"] >= 3, "ripple2b": lambda p: p["ripple2b"], "ripple3b": lambda p: p["ripple3b"],
         "past0": lambda p: p["past0"]}

SPECIAL = [0, 1, P - 1, P, P + 1, ONES, ONES - 1, PRIME_DIFF - 1, PRIME_DIFF + 1, 2**3071]


def _structured(rnd):
    c = rnd.randrange(6)
    if c == 0:  # all ones with a few low or mid bits cleared
        x = ONES
        for _ in range(rnd.randrange(1, 4)):
            x &= ~(1 << rnd.choice([rnd.randrange(64), rnd.randrange(3072)]))
        return x
    if c == 1:  # alternating all-ones and zero limb blocks
        return sum((B256 - 1) << (256 * k) for k in range(rnd.randrange(2), 12, 2))
    if c == 2:  # (2^k - 1)(2^m + 1): long runs of ones
        k = rnd.randrange(1, 3072)
        return (2**k - 1) * (2**rnd.randrange(0, 3072 - k) + 1) % TOP
    if c == 3:
        return rnd.choice(SPECIAL)
    if c == 4:  # all ones but one limb block
        k = rnd.randrange(12)
        return ONES ^ (rnd.getrandbits(256) << (256 * k))
    return rnd.getrandbits(3072)


def edge_cases(seed=7, n_structured=160):
    """[(a, b, label)]: the special values paired with each other, structured pairs, and pairs built to take each rare path
    (at least three per flag of FLAGS).  Every pair is checked with `paths` (which asserts the model's invariants)."""
    rnd = random.Random(seed)
    cases = [(a, b, "special") for i, a in enumerate(SPECIAL) for b in SPECIAL[i:]]
    cases += [(_structured(rnd), _structured(rnd), "structured") for _ in range(n_structured)]
    # a = 2^3072 - 1: a * b = (b - 1) * 2^3072 + (2^3072 - b), so the first fold is 2^3072 + b * (PRIME_DIFF - 1) - PRIME_DIFF.
    # b just above m * 2^3072 / (PRIME_DIFF - 1) leaves that first fold's low part within m * PRIME_DIFF of 2^3072: a third round.
    for m in (1, 2, 3, 1000, PRIME_DIFF - 3):
        b = (m * TOP + PRIME_DIFF) // (PRIME_DIFF - 1)
        cases += [(ONES, b, "round3"), (b, ONES - rnd.randrange(4) * (m == 1), "round3")]
    # b = 1 + k * 2^254 (k small) makes the low half of a * b all ones above limb block 0 and its high half k * 2^254: the
    # first fold's low block carries into 11 all-ones blocks, and the second-round addition runs out of block 0
    for k in (1, 2, 3, 5):
        cases += [(ONES, 1 + k * 2**254, "ripple3b"), (1 + k * 2**(254 + 256 * rnd.randrange(1, 11)), ONES, "past0")]
    # a product whose phase-2 blocks are all ones except for a carry from below: a * b = 2^(256 j) * (2^(256 t) - 1) + small
    for j in (1, 5, 11):
        a = ONES >> (256 * (12 - j))  # 2^(256 j) - 1
        cases += [(a, a, "ripple2b"), (a, ONES, "ripple2b"), (ONES, ONES - rnd.randrange(1, 2**32), "ripple2b")]
    out = []
    for a, b, label in cases:
        a, b = a % TOP, b % TOP
        out.append((a, b, label, paths(a, b)))
    return out


def flag_counts(cases):
    return {name: sum(1 for c in cases if f(c[3])) for name, f in FLAGS.items()}
