"""GPU-less tests of the standardness rule bodies (csrc/kgv_standard.cuh, host build in tests/hostsim/hostsim_standard.cpp) against the CPU
restatement (oracle_standard.py): 10^5 random scripts biased toward the edges of every rule - truncated pushes, PUSHDATA1/2/4, OP_RETURN first
and elsewhere, multisig opcodes at position 0 and after OP_0, OP_1..OP_16 or a data push, small-int last pushes, non-push signature scripts,
class near-misses - dust values on both sides of the threshold and above 2^64 / 1000, and relay fees up to the overflow."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import oracle_standard as os_

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
CSRC = os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc")
U64 = 2**64 - 1


@pytest.fixture(scope="module")
def hs():
    src, out = os.path.join(HS, "hostsim_standard.cpp"), os.path.join(HS, "libhostsim_standard.so")
    hdrs = [os.path.join(CSRC, f) for f in ("kgv_standard.cuh", "kgv_script_std.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return ctypes.CDLL(out)


def push(d, rng):
    n = len(d)
    r = rng.random()
    if r < 0.1:
        return bytes([0x4c, n & 0xFF]) + d
    if r < 0.15:
        return bytes([0x4d]) + (n & 0xFFFF).to_bytes(2, "little") + d
    if r < 0.2:
        return bytes([0x4e]) + n.to_bytes(4, "little") + d
    return (bytes([n]) if 0 < n <= 75 else bytes([0x4c, n]) if n <= 255 else bytes([0x4d]) + n.to_bytes(2, "little")) + d


SIGOPS = [0xac, 0xad, 0xab, 0xae, 0xaf, 0xa9]


def piece(rng):
    r = rng.random()
    if r < 0.25:
        return push(rng.randbytes(rng.choice([0, 1, 2, 20, 32, 33, 65, 75, 76, 255, 256])), rng)
    if r < 0.4:
        return bytes([rng.choice([0x00, 0x4f] + list(range(0x51, 0x61)))])
    if r < 0.6:
        return bytes([rng.choice(SIGOPS)])
    if r < 0.7:
        return bytes([0x6a])
    if r < 0.8:  # a truncated push
        return rng.choice([bytes([rng.randrange(1, 76)]), b"\x4c", b"\x4d\x01", b"\x4e\x01\x00", b"\x4c\x09\x01", b"\x4d\x00\x01" + bytes(5), b"\x4e\xff\xff\xff\xff"])
    return bytes([rng.randrange(256)])


def redeem(rng):
    return b"".join(piece(rng) for _ in range(rng.randrange(0, 12)))


def near_miss(rng):
    base = rng.choice([bytes([0x20]) + rng.randbytes(32) + b"\xac", bytes([0x21]) + rng.randbytes(33) + b"\xab", b"\xaa\x20" + rng.randbytes(32) + b"\x87"])
    r = rng.random()
    if r < 0.4:
        return base
    if r < 0.7:
        k = rng.choice([0, 1, len(base) - 1])
        return base[:k] + bytes([base[k] ^ (1 << rng.randrange(8))]) + base[k + 1:]
    return base[:-1] if rng.random() < 0.5 else base + bytes([rng.randrange(256)])


def random_script(rng):
    r = rng.random()
    if r < 0.25:
        return near_miss(rng)
    if r < 0.55:  # a P2SH signature script: pushes ending with a redeem script (or a small int / a non-push)
        s = b"".join(push(rng.randbytes(rng.choice([0, 64, 65])), rng) for _ in range(rng.randrange(0, 3)))
        last = rng.random()
        if last < 0.7:
            s += push(redeem(rng), rng)
        elif last < 0.85:
            s += bytes([rng.choice([0x00, 0x4f] + list(range(0x51, 0x61)))])
        else:
            s += bytes([rng.choice([0x61, 0x76, 0xac, 0x6a])]) + push(redeem(rng), rng)
        return s
    return redeem(rng)


def _arena(scripts):
    arena = b"".join(scripts) + bytes(8)
    off = np.cumsum([0] + [len(s) for s in scripts[:-1]]).astype(np.uint64)
    ln = np.array([len(s) for s in scripts], dtype=np.uint32)
    return np.frombuffer(arena, np.uint8).copy(), off, ln


def test_scripts_match_the_oracle(hs):
    rng = random.Random(20261016)
    scripts = [random_script(rng) for _ in range(100_000)]
    ver = np.array([0 if rng.random() < 0.95 else rng.choice([1, 0x100]) for _ in scripts], dtype=np.uint16)
    arena, off, ln = _arena(scripts)
    out, ops = np.zeros(len(scripts), np.uint64), np.zeros(len(scripts), np.uint64)
    hs.hs_scripts(arena.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p), ln.ctypes.data_as(ctypes.c_void_p),
                  ver.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(scripts)), out.ctypes.data_as(ctypes.c_void_p), ops.ctypes.data_as(ctypes.c_void_p))
    classes, unsp, bounds = {}, 0, set()
    for k, s in enumerate(scripts):
        c, u, b = os_.script_class(int(ver[k]), s), os_.is_unspendable(s), os_.sig_op_count_upper_bound_p2sh(s)
        got = int(out[k])
        assert (got & 3, (got >> 2) & 1, got >> 8) == (c, int(u), b), (k, s.hex())
        assert int(ops[k]) == os_.sig_op_count_by_opcodes(*os_.parse_script(s)), (k, s.hex())
        classes[c] = classes.get(c, 0) + 1
        unsp += u
        bounds.add(b)
    assert len(classes) == 4 and 10_000 < unsp < 90_000 and {0, 1, 16, 20} <= bounds and max(bounds) > 15


def test_dust_matches_the_oracle(hs):
    rng = random.Random(7)
    scripts, values, fees = [], [], []
    for _ in range(100_000):
        s = rng.choice([near_miss(rng), random_script(rng), b"", b"\x6a", bytes(rng.randrange(0, 300))])
        fee = rng.choice([0, 1, 3, 1000, 5000, rng.randrange(2**64), U64, 2**63])
        size = 8 + 2 + 8 + len(s) + 148
        edge = -(-fee * 3 * size // 1000)  # the least value that is not dust
        v = rng.choice([edge - 1, edge, edge + 1, 0, rng.randrange(2**64), U64, U64 // 1000, U64 // 1000 + 1, os_.MAX_SOMPI])
        scripts.append(s); values.append(min(max(v, 0), U64)); fees.append(fee)
    arena, off, ln = _arena(scripts)
    v, f = np.array(values, dtype=np.uint64), np.array(fees, dtype=np.uint64)
    out = np.zeros(len(scripts), np.uint8)
    hs.hs_dust(arena.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p), ln.ctypes.data_as(ctypes.c_void_p), v.ctypes.data_as(ctypes.c_void_p),
               f.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(scripts)), out.ctypes.data_as(ctypes.c_void_p))
    exp = np.array([os_.is_transaction_output_dust(a, s, b) for a, s, b in zip(values, scripts, fees)], dtype=np.uint8)
    assert (out == exp).all(), np.nonzero(out != exp)[0][:5]
    assert 0.2 < exp.mean() < 0.8


def test_relay_fee_matches_the_oracle(hs):
    rng = random.Random(3)
    mass = [rng.choice([0, 1, 250, 999, 1000, 100_000, 100_001, rng.randrange(2**40), rng.randrange(2**64)]) for _ in range(20_000)]
    fee = [rng.choice([0, 1, 3, 1000, U64 // 100_000, U64 // 100_000 + 1, rng.randrange(2**64), U64]) for _ in mass]
    for r in os_.golden()["relay_fee"]["rows"]:
        mass.append(r["size"]); fee.append(r["minimum_relay_transaction_fee"])
    m, f = np.array(mass, dtype=np.uint64), np.array(fee, dtype=np.uint64)
    out, ok = np.zeros(len(mass), np.uint64), np.zeros(len(mass), np.uint8)
    hs.hs_min_fee(m.ctypes.data_as(ctypes.c_void_p), f.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(mass)), out.ctypes.data_as(ctypes.c_void_p),
                  ok.ctypes.data_as(ctypes.c_void_p))
    n_over = 0
    for k in range(len(mass)):
        try:
            e = os_.minimum_required_transaction_relay_fee(mass[k], fee[k])
            assert ok[k] == 1 and int(out[k]) == e, (mass[k], fee[k])
        except OverflowError:
            assert ok[k] == 0, (mass[k], fee[k])
            n_over += 1
    assert 0 < n_over < len(mass) // 2
