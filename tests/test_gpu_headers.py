"""kgv_hash_headers / kgv_validate_headers_in_isolation on the GPU against the C restatement (tests/oracle_pow/ok_pow.c) and the
reference's own header hashes: every header of the three DAG fixtures, nonces ground to pass easy targets, each isolation rule on mutated
headers, genesis-shaped headers, host against device pointers, batch splits, 10^5 generated headers, the proof-of-work matrix on
caller matrices, and malformed arena layouts."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import oracle_header as oh
from rusty_kaspa_b200 import KgvError
from rusty_kaspa_b200.headers import (HEADER_STATUS, HeaderBatch, HeaderRules, debug_pow_matrix, hash_headers,
                                      validate_headers_in_isolation)

pytestmark = pytest.mark.gpu
KAT = json.load(open(os.path.join(oh.GOLDEN, "pow_kat.json")))


@pytest.fixture(scope="module")
def ok():
    return oh.c_oracle()


def _same(got, want):
    res, hh, pw = got
    eres, ehh, epw, _ = want
    assert res.tobytes() == eres.tobytes()
    if hh is not None:
        assert hh.tobytes() == ehh.tobytes()
    if pw is not None:
        assert pw.tobytes() == epw.tobytes()


@pytest.mark.parametrize("fixture", oh.FIXTURES)
def test_fixture_hashes_and_verdicts(gpu_ctx, ok, fixture):
    params, hdrs = oh.fixture_headers(fixture)
    b = HeaderBatch.from_dicts(hdrs)
    hh, pre = hash_headers(gpu_ctx, b)
    assert [bytes(x) for x in hh] == [h["hash"] for h in hdrs]
    for skip in (False, True):
        rules = oh.fixture_rules(params, skip_pow=skip)
        want = oh.oracle_validate(ok, b, rules)
        assert pre.tobytes() == want[3].tobytes()
        _same(validate_headers_in_isolation(gpu_ctx, b, rules, want_hash=True, want_pow=True), want)
        res = want[0]
        # the DAGs were built with skip_proof_of_work: no header but genesis meets its own bits
        assert int(res["pow_passed"].sum()) == 1
        assert set(res["status"].tolist()) <= ({HEADER_STATUS["Ok"], HEADER_STATUS["WrongBlockVersion"]} if skip else
                                               {HEADER_STATUS["InvalidPoW"], HEADER_STATUS["WrongBlockVersion"]})


def test_fixture_parent_levels(gpu_ctx):
    """Every fixture block listed at parents_by_level[L >= 1] of a child has a computed level >= L."""
    for fixture in oh.FIXTURES:
        params, hdrs = oh.fixture_headers(fixture)
        res, _, _ = validate_headers_in_isolation(gpu_ctx, HeaderBatch.from_dicts(hdrs), oh.fixture_rules(params))
        level = {h["hash"]: int(res["level"][i]) for i, h in enumerate(hdrs)}
        for h in hdrs:
            for L, ps in enumerate(h["parents_by_level"][1:], start=1):
                assert all(level[p] >= L for p in ps if p in level)


def _ground(ok, hdrs, bits, n, seed=1):
    """n fixture headers with their bits set to `bits` and a nonce ground on the C restatement so that the PoW meets it."""
    out = []
    for h in hdrs[1:n + 1]:
        g = dict(h, bits=bits)
        b = HeaderBatch.from_dicts([g])
        nonce = ctypes.c_uint64()
        assert ok.ok_pow_grind(b.headers.ctypes.data, b.parents.ctypes.data, b.level_len.ctypes.data, seed, 1 << 16, ctypes.byref(nonce)) == 1
        out.append(dict(g, nonce=nonce.value))
    return out


def test_ground_nonces_pass(gpu_ctx, ok):
    params, hdrs = oh.fixture_headers(oh.FIXTURES[1])
    passing = _ground(ok, hdrs, 0x2000FFFF, 40)        # exponent 0x20: target 0xFFFF * 2^232
    failing = [dict(h, nonce=h["nonce"] + 1) for h in passing]
    b = HeaderBatch.from_dicts(passing + failing)
    rules = oh.fixture_rules(params, skip_pow=False)
    want = oh.oracle_validate(ok, b, rules)
    _same(validate_headers_in_isolation(gpu_ctx, b, rules, want_hash=True, want_pow=True), want)
    res = want[0]
    assert (res["status"][:40] == HEADER_STATUS["Ok"]).all() and (res["pow_passed"][:40] == 1).all()
    for i, h in enumerate(passing):  # the level follows the PoW value
        assert res["level"][i] == max(rules.max_block_level - int.from_bytes(want[2][i].tobytes(), "little").bit_length(), 0)
    # an incremented nonce is almost surely above the target again; whichever way it falls, the GPU agrees with the oracle
    assert (res["status"][40:] == HEADER_STATUS["InvalidPoW"]).sum() > 20


def test_rules_in_order(gpu_ctx, ok):
    params, hdrs = oh.fixture_headers(oh.FIXTURES[1])
    base = _ground(ok, hdrs, 0x2000FFFF, 1)[0]
    lvl0 = base["parents_by_level"][0]
    rules = oh.fixture_rules(params, skip_pow=False, now_ms=base["timestamp"], max_block_parents=len(lvl0))
    tol = rules.timestamp_deviation_tolerance * 1000
    origin = [lvl0[0], b"\xfe" * 32] + lvl0[2:] if len(lvl0) > 1 else [b"\xfe" * 32]
    cases = [
        ("base", base, HEADER_STATUS["Ok"]),
        ("bad pow", dict(base, bits=0x03000001), HEADER_STATUS["InvalidPoW"]),
        ("origin", dict(base, parents_by_level=[origin] + base["parents_by_level"][1:], bits=0x03000001), HEADER_STATUS["OriginParent"]),
        ("too many", dict(base, parents_by_level=[lvl0 + [bytes(32)]] + base["parents_by_level"][1:], bits=0x03000001),
         HEADER_STATUS["TooManyParents"]),
        ("no parents", dict(base, parents_by_level=[[]] + base["parents_by_level"][1:], bits=0x03000001), HEADER_STATUS["NoParents"]),
        ("at the time limit", dict(base, timestamp=base["timestamp"] + tol, bits=0x03000001), HEADER_STATUS["InvalidPoW"]),
        ("future", dict(base, timestamp=base["timestamp"] + tol + 1, parents_by_level=[[]]), HEADER_STATUS["TimeTooFarIntoTheFuture"]),
        ("version", dict(base, version=2, timestamp=base["timestamp"] + tol + 1, parents_by_level=[[]]), HEADER_STATUS["WrongBlockVersion"]),
        ("genesis-shaped", dict(base, parents_by_level=[]), HEADER_STATUS["NoParents"]),
        ("genesis-shaped, old version", dict(base, parents_by_level=[], version=0), HEADER_STATUS["WrongBlockVersion"]),
    ]
    b = HeaderBatch.from_dicts([c[1] for c in cases])
    want = oh.oracle_validate(ok, b, rules)
    got = validate_headers_in_isolation(gpu_ctx, b, rules, want_hash=True, want_pow=True)
    _same(got, want)
    res = got[0]
    for i, (name, h, st) in enumerate(cases):
        assert res["status"][i] == st, name
    i = [c[0] for c in cases].index("too many")
    assert (res["a"][i], res["b"][i]) == (len(lvl0) + 1, len(lvl0))
    i = [c[0] for c in cases].index("future")
    assert (res["a"][i], res["b"][i]) == (base["timestamp"] + tol + 1, base["timestamp"] + tol)
    i = [c[0] for c in cases].index("version")
    assert res["a"][i] == 2
    for i in (8, 9):  # genesis: max level, passed
        assert res["level"][i] == rules.max_block_level and res["pow_passed"][i] == 1
    # with skip_pow the insufficient PoW is no longer an error; nothing else changes
    skip = oh.fixture_rules(params, skip_pow=True, now_ms=base["timestamp"], max_block_parents=len(lvl0))
    res2 = validate_headers_in_isolation(gpu_ctx, b, skip)[0]
    for i in range(len(cases)):
        assert res2["status"][i] == (HEADER_STATUS["Ok"] if res["status"][i] == HEADER_STATUS["InvalidPoW"] else res["status"][i]), cases[i][0]
    assert (res2["level"] == res["level"]).all()


def _random_headers(n, seed):
    rng = random.Random(seed)
    pool = [rng.randbytes(32) for _ in range(512)] + [b"\xfe" * 32]
    hs = []
    for _ in range(n):
        levels = []
        for L in range(rng.choice([0, 1, 1, 2, 3, 5, 10, 30])):
            levels.append(levels[-1] if L and rng.random() < 0.4 else [rng.choice(pool) for _ in range(rng.choice([0, 1, 1, 2, 3, 8, 17]))])
        e = rng.choice([0, 1, 2, 3, 4, 0x1D, 0x1F, 0x20, 0x20, 0x21, 0x22, 0x23, 0x40, 0xFF])
        hs.append({"version": rng.choice([1, 1, 1, 0, 2, 0xFFFF]), "parents_by_level": levels, "hash_merkle_root": rng.randbytes(32),
                   "accepted_id_merkle_root": rng.randbytes(32), "utxo_commitment": rng.randbytes(32),
                   "timestamp": rng.choice([rng.getrandbits(41), rng.getrandbits(64), 0]), "bits": (e << 24) | rng.getrandbits(24),
                   "nonce": rng.getrandbits(64), "daa_score": rng.getrandbits(rng.choice([8, 40, 64])),
                   "blue_score": rng.getrandbits(rng.choice([8, 40, 64])), "blue_work": rng.getrandbits(rng.choice([0, 1, 8, 70, 192])),
                   "pruning_point": rng.randbytes(32)})
    return hs


@pytest.fixture(scope="module")
def big():
    return HeaderBatch.from_dicts(_random_headers(100_000, 11))


RANDOM_RULES = dict(timestamp_deviation_tolerance=132, now_ms=1 << 41, block_version=1, max_block_parents=10, max_block_level=225)


def test_random_batch_matches_oracle(gpu_ctx, ok, big):
    for skip in (False, True):
        rules = HeaderRules(skip_pow=skip, **RANDOM_RULES)
        want = oh.oracle_validate(ok, big, rules)
        _same(validate_headers_in_isolation(gpu_ctx, big, rules, want_hash=True, want_pow=True), want)
        hh, pre = hash_headers(gpu_ctx, big)
        assert hh.tobytes() == want[1].tobytes() and pre.tobytes() == want[3].tobytes()
        if not skip:
            assert len(set(want[0]["status"].tolist())) == 7 and want[0]["pow_passed"].sum() > 1000


def _sub(b, lo, hi):
    return HeaderBatch(b.headers[lo:hi], b.level_len, b.parents)


def test_batch_splits_and_pointer_kinds(gpu_ctx, big):
    import torch
    rules = HeaderRules(**RANDOM_RULES)
    full = validate_headers_in_isolation(gpu_ctx, big, rules, want_hash=True, want_pow=True)
    for size in (1, 2, 2 * 132, 1000):
        parts = [validate_headers_in_isolation(gpu_ctx, _sub(big, lo, min(lo + size, 5000)), rules, want_hash=True, want_pow=True)
                 for lo in range(0, 5000, size)]
        for k in range(3):
            assert np.concatenate([p[k] for p in parts]).tobytes() == full[k][:5000].tobytes(), size
    # device pointers: the same call on torch tensors
    n = len(big)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    dh, dp, dl = dev(big.headers), dev(big.parents), dev(big.level_len)
    dres, dhash, dpow = (torch.zeros(n * k, dtype=torch.uint8, device="cuda") for k in (24, 32, 32))
    lib = gpu_ctx._lib
    gpu_ctx._check(lib.kgv_validate_headers_in_isolation(gpu_ctx._h, dh.data_ptr(), n, dp.data_ptr(), len(big.parents), dl.data_ptr(), len(big.level_len),
                                                         ctypes.byref(rules), dres.data_ptr(), dhash.data_ptr(), dpow.data_ptr()))
    assert dres.cpu().numpy().tobytes() == full[0].tobytes()
    assert dhash.cpu().numpy().tobytes() == full[1].tobytes() and dpow.cpu().numpy().tobytes() == full[2].tobytes()
    dpre = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    gpu_ctx._check(lib.kgv_hash_headers(gpu_ctx._h, dh.data_ptr(), n, dp.data_ptr(), len(big.parents), dl.data_ptr(), len(big.level_len),
                                        dhash.data_ptr(), dpre.data_ptr()))
    hh, pre = hash_headers(gpu_ctx, big)
    assert dhash.cpu().numpy().tobytes() == hh.tobytes() and dpre.cpu().numpy().tobytes() == pre.tobytes()
    # a device arena range outside the arena is reported as well
    bad = big.headers[:4].copy()
    bad["levels_off"][2] = len(big.level_len)
    bad["n_levels"][2] = 1
    with pytest.raises(KgvError):
        gpu_ctx._check(lib.kgv_hash_headers(gpu_ctx._h, dev(bad).data_ptr(), 4, dp.data_ptr(), len(big.parents), dl.data_ptr(), len(big.level_len),
                                            dhash.data_ptr(), None))


def test_malformed_layouts_are_refused(gpu_ctx, big):
    rules = HeaderRules(**RANDOM_RULES)
    h0 = big.headers
    k = next(i for i in range(len(h0)) if big.level_len[int(h0["levels_off"][i]):int(h0["levels_off"][i]) + int(h0["n_levels"][i])].sum() > 0)
    for field, value in (("levels_off", len(big.level_len)), ("parents_off", len(big.parents)), ("parents_off", 2**64 - 1),
                         ("levels_off", 2**32 - 1)):
        h = big.headers[k:k + 1].copy()
        h[field] = value
        b = HeaderBatch(h, big.level_len, big.parents)
        with pytest.raises(KgvError):
            validate_headers_in_isolation(gpu_ctx, b, rules)
        with pytest.raises(KgvError):
            hash_headers(gpu_ctx, b)
    # the context still works afterwards
    res = validate_headers_in_isolation(gpu_ctx, _sub(big, 0, 10), rules)[0]
    assert res.tobytes() == validate_headers_in_isolation(gpu_ctx, _sub(big, 0, 10), rules)[0].tobytes()


def test_device_rank_and_generate(gpu_ctx):
    mats = [c["matrix"] for c in KAT["compute_rank"]]
    want = [c["rank"] for c in KAT["compute_rank"]]
    full = KAT["generate_matrix"]["matrix"]
    mats += [[list(full[1])] + [list(r) for r in full[1:]], full, KAT["heavy_hash"]["matrix"], [[0] * 64] * 63 + [[1] * 64]]
    want += [63, 64, oh.compute_rank(KAT["heavy_hash"]["matrix"]), 1]
    ranks = debug_pow_matrix(gpu_ctx, 0, np.array(mats, dtype=np.uint16), len(mats))
    assert ranks.tolist() == want
    rng = random.Random(3)
    seeds = [bytes.fromhex(KAT["generate_matrix"]["seed"])] + [rng.randbytes(32) for _ in range(63)]
    m, tries = debug_pow_matrix(gpu_ctx, 1, np.frombuffer(b"".join(seeds), dtype=np.uint8), len(seeds))
    assert m[0].tolist() == full and tries[0] == 1
    for i in (1, 30, 63):
        pm, pt = oh.generate_matrix(seeds[i])
        assert m[i].tolist() == pm and tries[i] == pt
