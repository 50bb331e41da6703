"""GPU: the eight-lane field product and squaring (kgv_debug_selftest ops 12 and 13) against the bit-exact model in
tests/lanes_model.py, Python integers and the per-thread fe_mul / fe_sqr (ops 2 and 3)."""
import random

import pytest

import lanes_model as lm

pytestmark = pytest.mark.gpu
P, M = lm.P, 2**256
C = M - P


def _operands():
    rnd = random.Random(12)
    edge = [0, 1, 2, P - 1, P, P + 1, P + C - 1, M - 1, M - 2, M - C, 2**255, 2**224 - 1, 0xFFFFFFFF,
            sum(0xFFFFFFFF << (64 * i) for i in range(4))]
    a = [rnd.choice(edge) if rnd.random() < 0.3 else rnd.getrandbits(256) for _ in range(600)]
    b = [rnd.choice(edge) if rnd.random() < 0.3 else rnd.getrandbits(256) for _ in range(600)]
    cases, _ = lm.carry_cases()
    a += [x for x, _ in cases]
    b += [y for _, y in cases]
    # products landing next to 0, p and 2^256 (t or t + p is what the carries resolve to), and operands in [p, 2^256)
    for t in (0, 1, C - 1, C, P - 1, P - C, 2**32 - 1, 2**224):
        for _ in range(16):
            x = rnd.randrange(1, P)
            y = t * pow(x, -1, P) % P
            a.append(x + P if x < C else x)
            b.append(y + P if y < C else y)
    a.append(P - 1)
    b.append(P - 1)
    return a, b


def test_lane_mul_sqr_match_model_and_per_thread(gpu_ctx):
    a, b = _operands()
    for op, per_thread, f in ((12, 2, lambda x, y: (x, y)), (13, 3, lambda x, y: (x, x))):
        got = gpu_ctx.debug_selftest(op, a, b)
        ref = gpu_ctx.debug_selftest(per_thread, a, b)
        for g, r, x, y in zip(got, ref, a, b):
            u, v = f(x, y)
            assert g == lm.mul_lanes(u, v)[0], (op, hex(x), hex(y), hex(g))
            assert g < M and g % P == u * v % P == r % P
