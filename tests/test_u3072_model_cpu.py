"""The MuHash field product's host build (tests/hostsim, g++ over kgv_u3072.cuh) against the bit-exact model in
tests/u3072_model.py: both multipliers return exactly fold(a * b), and the crafted operands reach every rare path the GPU test
(tests/test_gpu_u3072.py) then runs through the device kernels."""
import ctypes
import random

import u3072_model as um
from test_hostsim import _build

W = ctypes.c_uint32 * 96


def _arr(v):
    return W(*[(v >> (32 * i)) & 0xFFFFFFFF for i in range(96)])


def _val(r):
    return sum(int(x) << (32 * i) for i, x in enumerate(r))


def test_model_fold_is_exact_for_both_host_multipliers():
    L = _build("hostsim_u3072")
    rnd = random.Random(4)
    cases = [(a, b) for a, b, _, _ in um.edge_cases()] + [(rnd.getrandbits(3072), rnd.getrandbits(3072)) for _ in range(40)]
    for a, b in cases:
        want = um.fold(a * b)
        assert want < 2**3072 and want % um.P == a * b % um.P
        r = W()
        L.hs_u3072_mul_mod(_arr(a), _arr(b), r, None)
        assert _val(r) == want, (hex(a), hex(b))
        r = W()
        assert L.hs_u3072_coop_mul_mod(_arr(a), _arr(b), r) == 0  # the top column's carry limb is empty
        assert _val(r) == want, (hex(a), hex(b))


def test_edge_cases_reach_every_rare_path():
    counts = um.flag_counts(um.edge_cases())
    assert all(c >= 4 for c in counts.values()), counts
    # the constructions do what their comments say
    b = (2**3072 + um.PRIME_DIFF) // (um.PRIME_DIFF - 1)
    assert um.paths(um.ONES, b)["rounds"] == 3
    assert um.paths(um.ONES, 1 + 2**254)["ripple3b"] and um.paths(um.ONES, 1 + 2**254)["past0"]
    # random operands take none of them
    rnd = random.Random(8)
    for _ in range(50):
        p = um.paths(rnd.getrandbits(3072), rnd.getrandbits(3072))
        assert p["rounds"] <= 2 and not any(f(p) for f in um.FLAGS.values())
