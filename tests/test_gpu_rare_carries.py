"""GPU: the rare carry / borrow propagation of fe_add and fe_sub (the 5-limb tails inc_hi5 / dec_hi5, and the second wrap
past 2^256) with operands built to reach them.  Random operands reach them with probability ~2^-32, so the PTX bodies of
those tails need explicit cases."""
import pytest

import pyref

pytestmark = pytest.mark.gpu
P, M = pyref.P, 2**256
C = M - P  # 2^32 + 977


def _cases():
    add = [(M - 1, M - 1), (M - 1, 1), (M - 1, C), (M - C, M - 1), ((M - 1) ^ (1 << 100), M - 1 - (1 << 20)),
           (M - 2**96, 2**96 - 1), (M - 2**96 + 5, M - 7), (M - 2**200, M - 2**96 + 3)]
    sub = [(0, M - 1), (0, 1), (1, M - 1), (C - 1, M - 1), (2**96, 2**96 + 1), (5, M - 2**96), (2**200, 2**200 + C),
           (0, C), (C, M - 1)]
    return add, sub


def test_fe_add_sub_rare_propagation(gpu_ctx):
    add, sub = _cases()
    for op, cases, f in ((8, add, lambda x, y: x + y), (9, sub, lambda x, y: x - y)):
        a, b = [x for x, _ in cases], [y for _, y in cases]
        for got, x, y in zip(gpu_ctx.debug_selftest(op, a, b), a, b):
            assert got < M and got % P == f(x, y) % P, (op, hex(x), hex(y))
