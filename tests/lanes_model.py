"""Bit-exact model of the eight-lane field product (fe_mul_lanes, rusty_kaspa_b200/csrc/kgv_lanes.cuh).

The device code keeps one limb per lane and resolves carries in rounds of shuffles and one carry-lookahead vote; its rare
paths are a carry rippling through lanes whose limb is all ones, and the sum wrapping past 2^256.  Random operands reach a
long ripple with probability about 2^-31, so `carry_cases` searches structured operands for pairs that reach each path,
and the model reports which paths a pair took.  The GPU test compares the device's limbs with `mul_lanes` exactly.
"""
import random

P = 2**256 - 2**32 - 977
M32 = 0xFFFFFFFF


def _limbs(x):
    return [(x >> (32 * i)) & M32 for i in range(8)]


def mul_lanes(a, b):
    """(result, paths) of fe_mul_lanes(a, b).  paths: 'ripple' = the longest run of lanes a lookahead carry entered
    (0 = none), 'wrap' = the sum wrapped past 2^256, 'g0' = lane 0 generated a carry."""
    A, B = _limbs(a), _limbs(b)
    L, H = [0] * 8, [0] * 8
    for k in range(8):
        for s in range(8):
            if s <= k:
                L[k] += A[(k - s) % 8] * B[s]
            else:
                H[k] += A[(k - s) % 8] * B[s]
    assert H[7] == 0
    z = [L[k] + 977 * H[k] + (H[k - 1] if k else 0) for k in range(8)]
    assert max(z) < 2**78
    z0, z1, z2 = [v & M32 for v in z], [(v >> 32) & M32 for v in z], [v >> 64 for v in z]
    x = []
    for k in range(8):
        v = z0[k] + (1 if k >= 1 else 977) * z1[(k - 1) % 8] + (1 if k >= 2 else 977) * z2[(k - 2) % 8]
        v += (z1[7] + z2[6]) if k == 1 else z2[7] if k == 2 else 0
        x.append(v)
    assert max(x) < 2**43
    xh = [v >> 32 for v in x]
    y = [(x[k] & M32) + (977 if k == 0 else 1) * xh[(k - 1) % 8] + (xh[7] if k == 1 else 0) for k in range(8)]
    assert max(y) < 2**33
    v = [t & M32 for t in y]
    g = [t >> 32 for t in y]
    paths = {"ripple": 0, "wrap": False, "g0": bool(g[0])}

    def ripple(v, g):
        G = sum(g[k] << k for k in range(8))
        assert not any(g[k] and v[k] == M32 for k in range(8))
        X = G | sum((v[k] == M32) << k for k in range(8))
        S = X + G
        cin = S ^ X ^ G
        run = best = 0
        for k in range(8):
            run = run + 1 if (cin >> k) & 1 else 0
            best = max(best, run)
        paths["ripple"] = max(paths["ripple"], best)
        return [(v[k] + ((cin >> k) & 1)) & M32 for k in range(8)], S >> 8

    v, wrap = ripple(v, g)
    if wrap:
        paths["wrap"] = True
        t = [v[0] + 977, v[1] + 1] + v[2:]
        v, again = ripple([u & M32 for u in t], [u >> 32 for u in t])
        assert not again
    r = sum(v[k] << (32 * k) for k in range(8))
    assert r % P == a * b % P
    return r, paths


def carry_cases(seed=5, tries=40000):
    """Operand pairs, some random and some built from structured limbs, that together reach every rare path of
    fe_mul_lanes: a lookahead carry through all eight lanes, a wrap past 2^256, a carry generated at lane 0."""
    rnd = random.Random(seed)
    special = [0, 1, 2, 977, 0x3D1, 2**31, M32, M32 - 1, M32 - 977, 0xFFFFFC2F, 0xFFFFFFFE]
    want = {"ripple8": None, "ripple7": None, "wrap": None, "g0": None, "wrap_ripple": None}
    base = [(2**256 - 1, 2**256 - 1), (P - 1, P - 1), (P, P), (P + 1, 2**256 - 1), (2**256 - 1, 1), (P - 1, 2)]
    for _ in range(tries):
        if all(want.values()):
            break
        a = sum((rnd.choice(special) if rnd.random() < 0.8 else rnd.getrandbits(32)) << (32 * i) for i in range(8))
        j = rnd.randrange(8)
        b = rnd.choice([1, 2, 977, M32, 2**32 + 977, rnd.getrandbits(32)]) << (32 * j)
        if rnd.random() < 0.3:
            b += rnd.choice([0, 1, M32]) << (32 * rnd.randrange(8))
        b %= 2**256
        _, p = mul_lanes(a, b)
        key = ("wrap_ripple" if p["wrap"] and p["ripple"] >= 4 else None, "ripple8" if p["ripple"] >= 8 else None,
               "ripple7" if p["ripple"] >= 7 else None, "wrap" if p["wrap"] else None, "g0" if p["g0"] else None)
        for kname in key:
            if kname and want[kname] is None:
                want[kname] = (a, b)
    missing = [k for k, v in want.items() if v is None]
    return base + [v for v in want.values() if v is not None], missing
