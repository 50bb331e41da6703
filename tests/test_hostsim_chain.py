"""GPU-less test of the coinbase builder of kgv_replay_verify_chain (csrc/kgv_chain.cuh, host build in tests/hostsim/hostsim_chain.cpp)
against the CPU restatement of expected_coinbase_transaction (oracle_chain.py): 10^4 random mergesets with blues, reds, non-DAA blues and
reds, zero rewards, miner scripts up to the 150-byte maximum, large extra data, mergesets past 32 blocks, and subsidy + fee sums and red sums
at and one past u64::MAX.  Every case must give the same expected-coinbase hash, or the same panic status."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import oracle_body as ob
import oracle_chain as oc
import pyref

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
CSRC = os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc")
U64 = 2**64 - 1
MAX_PAYLOAD_LEN, MAX_SPK_LEN = 204, 150


@pytest.fixture(scope="module")
def hs():
    src, out = os.path.join(HS, "hostsim_chain.cpp"), os.path.join(HS, "libhostsim_chain.so")
    hdrs = [os.path.join(CSRC, f) for f in ("kgv_chain.cuh", "kgv_txhash.cuh", "kgv_blake2b.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    lib = ctypes.CDLL(out)
    lib.hs_expected_coinbase.restype = ctypes.c_uint32
    lib.hs_expected_coinbase.argtypes = [ctypes.c_uint32] + [ctypes.c_void_p] * 7 + [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint32,
                                                                                     ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p]
    lib.hs_payload_parse.restype = ctypes.c_uint32
    lib.hs_payload_parse.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint64]
    return lib


def _amount(rng):
    r = rng.random()
    if r < 0.2:
        return 0
    if r < 0.3:
        return U64 - rng.randrange(0, 3)
    if r < 0.4:
        return 2**63 + rng.randrange(0, 3)
    return rng.randrange(0, 50_000_000_000)


def _mergeset(rng):
    n = rng.choice([0, 1, 2, 3, 5, 8, 17, 33, 40])
    out = []
    for _ in range(n):
        sub, fees = _amount(rng), _amount(rng)
        if rng.random() < 0.1:  # a sum exactly at u64::MAX, or one past it
            fees = U64 - sub + rng.randrange(0, 2) if sub else U64
        script = rng.randbytes(rng.choice([0, 1, 34, 35, 149, 150]))
        flags = rng.choice([0, 0, 0, oc.RED, oc.NON_DAA, oc.RED | oc.NON_DAA])
        out.append((sub, min(fees, U64), rng.randrange(0, 3), script, flags))
    return out


def _miner_payload(rng):
    script = rng.randbytes(rng.choice([0, 34, 35, 150]))
    extra = rng.randbytes(rng.randrange(0, MAX_PAYLOAD_LEN - 19 - len(script) + 1))
    p = ob.coinbase_payload(rng.randrange(0, 2**40), rng.randrange(0, 2**40), script, rng.randrange(0, 3), extra)
    r = rng.random()
    if r < 0.03:
        p = p[:rng.randrange(0, 19)]  # below the minimum length
    elif r < 0.06:
        p = p + bytes(MAX_PAYLOAD_LEN + 1 - len(p))  # above the maximum length
    elif r < 0.08 and len(script) > 0:
        p = p[:19 + len(script) - 1]  # cannot contain its script
    return p


def test_expected_coinbase_matches_the_restatement(hs):
    rng = random.Random(2024)
    seen = {}
    for case in range(10_000):
        rewards = _mergeset(rng)
        miner = _miner_payload(rng)
        blue, subsidy = rng.randrange(0, 2**50), rng.choice([0, 1, 44_000_000_000, U64])
        n = len(rewards)
        arena = b"".join(r[3] for r in rewards) + b"\0"
        off = np.cumsum([0] + [len(r[3]) for r in rewards[:-1]]).astype(np.uint32) if n else np.zeros(1, np.uint32)
        arr = lambda v, t: np.array(v if v else [0], dtype=t)
        sub, fees = arr([r[0] for r in rewards], np.uint64), arr([r[1] for r in rewards], np.uint64)
        flags, ln, ver = arr([r[4] for r in rewards], np.uint8), arr([len(r[3]) for r in rewards], np.uint32), arr([r[2] for r in rewards], np.uint16)
        abuf = np.frombuffer(arena, dtype=np.uint8).copy()
        out = np.zeros(32, dtype=np.uint8)
        st = hs.hs_expected_coinbase(n, sub.ctypes.data, fees.ctypes.data, flags.ctypes.data, abuf.ctypes.data, off.ctypes.data, ln.ctypes.data, ver.ctypes.data,
                                     blue, subsidy, miner, len(miner), MAX_PAYLOAD_LEN, MAX_SPK_LEN, out.ctypes.data)
        try:
            exp = pyref.tx_hash(oc.expected_coinbase_transaction(rewards, blue, subsidy, miner, MAX_PAYLOAD_LEN, MAX_SPK_LEN))
            assert st == 0 and out.tobytes() == exp, (case, st, rewards, miner.hex())
        except oc.ChainPanic as p:
            assert st == p.status, (case, st, p.status, rewards)
        seen[st] = seen.get(st, 0) + 1
    assert seen.get(0, 0) > 3000 and seen.get(oc.STATUS["RewardOverflow"], 0) > 500 and seen.get(oc.STATUS["CoinbasePayloadUnparsable"], 0) > 200, seen


def test_payload_parse_matches_the_restatement(hs):
    rng = random.Random(7)
    for _ in range(3000):
        p = _miner_payload(rng)
        if rng.random() < 0.2:
            p = p[:18] + bytes([rng.randrange(256)]) + p[19:]  # any script length byte
        try:
            ob.deserialize_coinbase_payload(p, MAX_PAYLOAD_LEN, MAX_SPK_LEN)
            want = 0
        except ob.BodyError as e:
            want = e.verdict["tx_status"]
        assert hs.hs_payload_parse(p, len(p), MAX_PAYLOAD_LEN, MAX_SPK_LEN) == want
