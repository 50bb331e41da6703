"""The eight-lane field product's carry schedule (tests/lanes_model.py, a bit-exact model of fe_mul_lanes) against Python
integers: the bounds each round relies on hold, the result is weakly reduced and congruent to the product, and the
crafted operands reach the rare paths the GPU test then runs on the device."""
import random

import lanes_model as lm

P, M = lm.P, 2**256


def test_model_random_and_edges():
    rnd = random.Random(3)
    edge = [0, 1, 2, P - 1, P, P + 1, M - 1, M - 2**32, 2**255, 2**224 - 1, 0xFFFFFFFF]
    pairs = [(x, y) for x in edge for y in edge] + [(rnd.getrandbits(256), rnd.getrandbits(256)) for _ in range(3000)]
    for a, b in pairs:
        r, _ = lm.mul_lanes(a, b)  # asserts the round bounds and r == a*b mod p
        assert 0 <= r < M


def test_carry_cases_reach_rare_paths():
    cases, _ = lm.carry_cases()
    paths = [lm.mul_lanes(a, b)[1] for a, b in cases]
    assert any(p["wrap"] for p in paths)
    assert any(p["g0"] for p in paths)
    assert any(p["wrap"] and p["ripple"] >= 5 for p in paths)
    assert max(p["ripple"] for p in paths) >= 5
