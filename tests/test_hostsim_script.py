"""GPU-less tests of the DEVICE script engine (csrc/kgv_script_dev.cuh, host build in tests/hostsim/hostsim_script.cpp), driven round by
round as kgv_scripts_dev.cu drives it (run from the start over the verdict log, answer the one request, repeat), against the host engine
of libkgv.so (kgv_script_execute), which the reference's own corpus pins (tests/test_host_vm.py):
  * the 850 corpus rows and the mainnet KATs, with verdicts from the CPU oracle;
  * 10^5 seeded random scripts from a weighted grammar, each compared with the host engine for an identical ScriptErr (both engines get
    the same deterministic stand-in verdicts, parse errors included, so the control flow after every kind of verdict is compared);
  * the scratch bounds: 244-item stacks, 201 hashing opcodes in a bare spk and in a redeem script, 201-deep IF nesting, 10 000-byte
    scripts and the most signature checks one input can make."""
import copy
import ctypes
import hashlib
import os
import random
import subprocess

import numpy as np
import pytest

from golden_util import entry_from_json, load, tx_from_json
from rusty_kaspa_b200 import _lib
from rusty_kaspa_b200.txbatch import build_batch
from rusty_kaspa_b200.validator import SCRIPT_ERR_NAMES, script_execute
from rusty_kaspa_b200.verifier import _c_batch
from test_host_vm import RESULT_NAMES, oracle_verdicts, spending_tx

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
CSRC = os.path.join(HS, "..", "..", "rusty_kaspa_b200", "csrc")
NEEDS = 254
U64_MAX = 2**64 - 1


@pytest.fixture(scope="module")
def se():
    src, out = os.path.join(HS, "hostsim_script.cpp"), os.path.join(HS, "libhostsim_script.so")
    hdrs = [os.path.join(CSRC, f) for f in ("kgv_script_dev.cuh", "kgv_txhash.cuh", "kgv_blake2b.cuh", "kgv_sha256.cuh", "kgv_script_std.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs + [src]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    lib = ctypes.CDLL(out)
    lib.hs_script_run.restype = ctypes.c_int
    lib.hs_compare.restype = ctypes.c_int
    return lib


class _Req:
    def __init__(self, raw, tx, in_abs):
        self.hash_type, self.ecdsa = raw[0], raw[1]
        self.key_len = 33 if raw[1] else 32
        self.key, self.sig = bytes(raw[2:35]), bytes(raw[35:99])
        self.tx, self.input = tx, in_abs


def dev_execute(se, batch, tx, k, verdict):
    """the device engine's result for one input, verdicts from `verdict(request)` (the host engine's request interface)"""
    cb = _c_batch(batch, with_entries=True)
    vs, raw = [], (ctypes.c_uint8 * 99)()
    in_abs = int(batch.txs[tx]["first_input"]) + k
    for _ in range(260):
        arr = (ctypes.c_uint8 * max(1, len(vs)))(*vs)
        r = se.hs_script_run(ctypes.byref(cb), tx, k, arr, len(vs), raw)
        if r != NEEDS:
            return r
        vs.append(int(verdict(_Req(bytes(raw), tx, in_abs))))
    raise AssertionError("more than 259 rounds")


def compare(se, batch, mode=0):
    lib = _lib.load()
    cb = _c_batch(batch, with_entries=True)
    n = len(batch.inputs)
    dev, host, checks = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint32)
    fn = ctypes.cast(lib.kgv_script_execute, ctypes.c_void_p)
    assert se.hs_compare(ctypes.byref(cb), fn, mode, dev.ctypes.data, host.ctypes.data, checks.ctypes.data) == 0
    return dev, host, checks


def test_reference_script_corpus(se, oracle):
    rows = load("script_tests.json.gz")["rows"]
    failures, seen = [], set()
    for i, r in enumerate(rows):
        if "builder_error" in r:
            continue
        tx, entries = spending_tx(bytes.fromhex(r["sigscript"]), bytes.fromhex(r["spk"]))
        b = build_batch([tx], [entries])
        got = dev_execute(se, b, 0, 0, oracle_verdicts(oracle, b))
        name = SCRIPT_ERR_NAMES[got]
        seen.add(name)
        if r["expected"] not in RESULT_NAMES.get(name, []) or got != script_execute(b, 0, 0, oracle_verdicts(oracle, b)):
            failures.append((i, r["sig_text"][:60], r["spk_text"][:60], r["expected"], name))
    assert not failures, failures[:10]
    assert len(seen) >= 20


def test_mainnet_kats(se, oracle):
    for c in load("check_scripts_kat.json")["cases"]:
        tx, entries = tx_from_json(c["tx"]), [entry_from_json(e) for e in c["entries"]]
        tx2 = copy.deepcopy(tx)
        tx2["inputs"].append(copy.deepcopy(tx2["inputs"][-1]))
        for t, e, exp in ((tx, entries, c["expected"]), (tx2, entries + [copy.deepcopy(entries[-1])], c["expected_duplicated_input"])):
            b = build_batch([t], [e])
            got = "Ok"
            for k in range(len(t["inputs"])):
                err = dev_execute(se, b, 0, k, oracle_verdicts(oracle, b))
                assert err == script_execute(b, 0, k, oracle_verdicts(oracle, b)), (c["name"], k)
                if err:
                    got = SCRIPT_ERR_NAMES[err]
                    break
            if exp == "AnyError":
                assert got != "Ok", c["name"]
            else:
                assert got == exp, (c["name"], got, exp)


# ---- the random script grammar
EDGE_NUMS = [0, 1, -1, 2, 16, 17, -16, 127, 128, -127, -128, 255, 256, 32767, 32768, -32768, 2**31 - 1, 2**31, -2**31, 2**32, 2**39,
             2**62, 2**63 - 1, -(2**63 - 1), 2**62 + 2**61, -(2**62 + 2**61), 500000000000, 500000000001, 2**63 + 5]
STACK_OPS = [0x6b, 0x6c, 0x6d, 0x6e, 0x6f, 0x70, 0x71, 0x72, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x7b, 0x7c, 0x7d, 0x82, 0x87, 0x88, 0x69, 0x61]
ARITH_OPS = [0x8b, 0x8c, 0x8f, 0x90, 0x91, 0x92, 0x93, 0x94, 0x9a, 0x9b, 0x9c, 0x9d, 0x9e, 0x9f, 0xa0, 0xa1, 0xa2, 0xa3, 0xa4, 0xa5]
INTRO_OPS = [0xb3, 0xb4, 0xb9, 0xbe, 0xbf, 0xc2, 0xc3]
ODD_OPS = [0x50, 0x62, 0x65, 0x66, 0x89, 0x8a, 0x7e, 0x95, 0x6a, 0xa6, 0xb2, 0xc4, 0xff, 0x67, 0x68]
HASH_TYPES = [1, 2, 4, 0x81, 0x82, 0x84, 1, 1, 0, 3, 0x83]


def num_bytes(x):
    if x == 0:
        return b""
    neg, p, out = x < 0, abs(x), bytearray()
    while p:
        out.append(p & 0xFF)
        p >>= 8
    if out[-1] & 0x80:
        out.append(0x80 if neg else 0)
    elif neg:
        out[-1] |= 0x80
    return bytes(out)


def push(data, rng):
    n = len(data)
    if rng.random() < 0.08:  # a non-minimal encoding
        return rng.choice([bytes([0x4C, n]) if n < 256 else bytes([0x4D]) + n.to_bytes(2, "little"), bytes([0x4E]) + n.to_bytes(4, "little")]) + data
    if n == 0:
        return b"\x00"
    if n == 1 and 1 <= data[0] <= 16:
        return bytes([0x50 + data[0]])
    if n == 1 and data[0] == 0x81:
        return b"\x4f"
    if n <= 75:
        return bytes([n]) + data
    if n <= 255:
        return bytes([0x4C, n]) + data
    return bytes([0x4D]) + n.to_bytes(2, "little") + data


def push_num(x, rng):
    b = num_bytes(x)
    if rng.random() < 0.05:
        b = b + b"\x00"  # not minimally encoded
    return push(b, rng)


def sig_item(rng):
    r = rng.random()
    if r < 0.1:
        return b""
    if r < 0.2:
        return rng.randbytes(rng.choice([1, 63, 64, 66, 70]))
    return rng.randbytes(64) + bytes([rng.choice(HASH_TYPES)])


def key_item(rng, ecdsa):
    r = rng.random()
    if r < 0.1:
        return rng.randbytes(rng.choice([0, 31, 33 if not ecdsa else 32, 65]))
    return rng.randbytes(33 if ecdsa else 32)


def fragment(rng, depth, n_in, n_out):
    r = rng.random()
    if r < 0.18:
        return push(rng.randbytes(rng.choice([0, 1, 2, 3, 8, 9, 20, 32, 75, 76, 255, 256, 520, 521])), rng)
    if r < 0.30:
        return push_num(rng.choice(EDGE_NUMS + [rng.randrange(-300, 300)]), rng)
    if r < 0.36:
        return bytes([rng.choice([0x00, 0x4F] + list(range(0x51, 0x61)))])
    if r < 0.48:
        return bytes([rng.choice(STACK_OPS)])
    if r < 0.58:
        return bytes([rng.choice(ARITH_OPS)])
    if r < 0.62:
        return bytes([rng.choice([0xA8, 0xAA])])
    if r < 0.67 and depth < 4:
        body = b"".join(fragment(rng, depth + 1, n_in, n_out) for _ in range(rng.randrange(0, 4)))
        alt = b"".join(fragment(rng, depth + 1, n_in, n_out) for _ in range(rng.randrange(0, 3)))
        cond = rng.choice([b"\x51", b"\x00", b"", b"\x52", push(b"\x01", rng)])
        tail = b"\x68" if rng.random() < 0.93 else b""
        return cond + bytes([rng.choice([0x63, 0x64])]) + body + (b"\x67" + alt if rng.random() < 0.5 else b"") + tail
    if r < 0.71:
        return push_num(rng.choice([0, 50, 100, 500000000000, 500000000001, 2**32, 2**63, -1]), rng) + bytes([rng.choice([0xB0, 0xB1])])
    if r < 0.78:
        op = rng.choice(INTRO_OPS)
        idx = b"" if op in (0xB3, 0xB4, 0xB9) else push_num(rng.choice([0, 1, n_in - 1, n_in, n_out, -1, 2**31]), rng)
        return idx + bytes([op])
    if r < 0.88:
        ecdsa = rng.random() < 0.3
        op = rng.choice([0xAB, 0xAB]) if ecdsa else rng.choice([0xAC, 0xAD])
        if ecdsa and rng.random() < 0.5:
            op = 0xAB
        return push(sig_item(rng), rng) + push(key_item(rng, ecdsa), rng) + bytes([op])
    if r < 0.93:
        ecdsa = rng.random() < 0.3
        nk = rng.choice([0, 1, 2, 3, 5, 20, 21])
        ns = rng.choice([0, 1, 2, min(nk, 3), nk + 1])
        sigs = b"".join(push(sig_item(rng), rng) for _ in range(max(0, ns)))
        keys = b"".join(push(key_item(rng, ecdsa), rng) for _ in range(max(0, nk)))
        op = 0xA9 if ecdsa else rng.choice([0xAE, 0xAF])
        return sigs + push_num(ns, rng) + keys + push_num(nk, rng) + bytes([op])
    if r < 0.97:
        return bytes([rng.choice(ODD_OPS)])
    return bytes([rng.randrange(256)]) + rng.randbytes(rng.randrange(0, 3))


def random_script(rng, n_in, n_out, length):
    return b"".join(fragment(rng, 0, n_in, n_out) for _ in range(length))


def random_tx(rng):
    n_in, n_out = rng.choice([1, 1, 2, 3]), rng.choice([1, 2])
    inputs, entries = [], []
    for _ in range(n_in):
        kind = rng.random()
        if kind < 0.3:  # P2SH: push-only sigscript ending with the redeem script
            redeem = random_script(rng, n_in, n_out, rng.randrange(1, 8))
            if rng.random() < 0.05:
                redeem = rng.choice([b"", b"\x51", b"\x00"])
            h = hashlib.blake2b(redeem, digest_size=32).digest()
            if rng.random() < 0.05:
                h = bytes(32)
            spk = b"\xaa\x20" + h + b"\x87"
            pre = b"".join(push(rng.randbytes(rng.choice([0, 1, 65, 66])), rng) for _ in range(rng.randrange(0, 3)))
            ss = pre + push(redeem, rng)
        else:
            spk = random_script(rng, n_in, n_out, rng.randrange(0, 10))
            ss = b"".join(fragment(rng, 3, n_in, n_out) if rng.random() < 0.1 else push(rng.randbytes(rng.choice([0, 1, 65, 33])), rng)
                          for _ in range(rng.randrange(0, 4)))
        inputs.append({"txid": rng.randbytes(32), "index": rng.randrange(4), "sigscript": ss, "sequence": rng.choice([0, 100, 2**63, U64_MAX, 2**32 + 7]),
                       "sig_op_count": rng.choice([0, 1, 2, 3, 20, 255])})
        entries.append({"amount": rng.choice([0, 10**9, 2**63 - 1, 2**63, U64_MAX]), "spk_version": 0 if rng.random() < 0.95 else 1, "script": spk,
                        "block_daa_score": 5, "is_coinbase": False})
    outputs = [{"value": rng.choice([0, 5, 2**63, 2**63 - 1]), "spk_version": rng.choice([0, 0, 1, 0x1234]), "script": rng.randbytes(rng.choice([0, 34, 35, 80]))}
               for _ in range(n_out)]
    tx = {"version": 0, "inputs": inputs, "outputs": outputs, "lock_time": rng.choice([0, 50, 100, 500000000000, 600000000000]),
          "subnetwork_id": bytes(20), "gas": 0, "payload": b"", "mass": 0}
    return tx, entries


def random_batches(seed, n_txs, per_batch=2000):
    rng = random.Random(seed)
    for lo in range(0, n_txs, per_batch):
        txs, ents = zip(*[random_tx(rng) for _ in range(min(per_batch, n_txs - lo))])
        yield build_batch(list(txs), list(ents))


def test_random_scripts_match_host_engine(se):
    n_inputs, errs, max_checks = 0, {}, 0
    for b in random_batches(20261016, 60_000):
        dev, host, checks = compare(se, b)
        bad = np.nonzero(dev != host)[0]
        assert len(bad) == 0, [(int(i), SCRIPT_ERR_NAMES.get(int(dev[i])), SCRIPT_ERR_NAMES.get(int(host[i]))) for i in bad[:5]]
        n_inputs += len(dev)
        for v in dev:
            errs[int(v)] = errs.get(int(v), 0) + 1
        max_checks = max(max_checks, int(checks.max()))
    assert n_inputs >= 100_000
    assert len(errs) >= 28, sorted(SCRIPT_ERR_NAMES[e] for e in errs)  # most error classes are reached
    assert errs.get(0, 0) > 1000 and max_checks >= 3


def _one_input_batch(ss, spk, sig_op_count=255, lock_time=0):
    tx = {"version": 0, "inputs": [{"txid": bytes(32), "index": 0, "sigscript": ss, "sequence": 0, "sig_op_count": sig_op_count}],
          "outputs": [{"value": 1, "spk_version": 0, "script": b"\x51"}], "lock_time": lock_time, "subnetwork_id": bytes(20), "gas": 0, "payload": b"", "mass": 0}
    return tx, [{"amount": 10, "spk_version": 0, "script": spk, "block_daa_score": 0, "is_coinbase": False}]


def p2sh(redeem, pre=b""):
    return pre + push(redeem, _Minimal()) if len(redeem) <= 520 else None, b"\xaa\x20" + hashlib.blake2b(redeem, digest_size=32).digest() + b"\x87"


class _Minimal:  # push() with this never picks a non-minimal encoding
    def random(self):
        return 1.0


def bound_cases():
    rng = _Minimal()
    k = b"\xaa" + bytes(31)  # mode 1: keys starting 0xAA verify
    kbad = b"\x01" + bytes(31)
    sig = push(bytes(64) + b"\x01", rng)
    h32 = push(bytes(range(32)), rng)
    cases = {
        "244 items": (b"\x51" * 244, b"\x6d" * 121 + b"\x75"),
        "245 items": (b"\x51" * 244, b"\x76"),
        "243 + 3DUP": (b"\x51" * 242, b"\x6f"),
        "alt stack full": (b"\x51" * 244, b"\x6b" * 122 + b"\x6c" * 122 + b"\x6d" * 121 + b"\x75"),
        "201 hashes bare": (b"", h32 + b"\xaa" * 100 + b"\xa8" * 101),
        "202 hashes bare": (b"", h32 + b"\xaa" * 202),
        "201 IF deep": (b"\x51" * 201, b"\x63" * 201),
        "100 IF deep balanced": (b"\x51" * 101, b"\x63" * 100 + b"\x68" * 100),
        "10000-byte spk": (b"", (b"\x4d\x08\x02" + bytes(520) + b"\x75") * 19 + b"\x29" + bytes(41) + b"\x75\x51"),
        "checks: 9 multisig + 11 checksig": (b"", (sig + b"\x51" + b"".join(push(kbad, rng) for _ in range(19)) + push(k, rng) + b"\x01\x14" + b"\xaf") * 9
                                              + (sig + push(k, rng) + b"\xad") * 11 + b"\x51"),
        "checks beyond sig_op_count": (b"", (sig + push(kbad, rng) + b"\xac\x75") * 60 + b"\x51"),
    }
    redeem = h32 + b"\xaa" * 100 + b"\xa8" * 101
    ss, spk = p2sh(redeem)
    cases["201 hashes in redeem"] = (ss, spk)
    ss, spk = p2sh(h32 + b"\xaa" * 202)
    cases["202 hashes in redeem"] = (ss, spk)
    ss, spk = p2sh(b"\x51" * 240 + b"\x6f")
    cases["redeem at the stack edge"] = (b"\x51" * 3 + ss, spk)
    cases["small-int redeem"] = (b"\x51" * 2 + b"\x51", b"\xaa\x20" + hashlib.blake2b(b"\x01", digest_size=32).digest() + b"\x87")
    return cases


def test_scratch_bounds_are_decided_and_match(se):
    cases = bound_cases()
    txs, ents = [], []
    for name, (ss, spk) in cases.items():
        t, e = _one_input_batch(ss, spk, sig_op_count=255 if "beyond" not in name else 50)
        txs.append(t); ents.append(e)
    txs.append(_one_input_batch(b"", b"\x51" * 10001)[0]); ents.append(_one_input_batch(b"", b"\x51" * 10001)[1])
    b = build_batch(txs, ents)
    dev, host, checks = compare(se, b, mode=1)
    names = list(cases) + ["10001-byte spk"]
    got = {n: (SCRIPT_ERR_NAMES[int(d)], int(c)) for n, d, c in zip(names, dev, checks)}
    assert (dev == host).all(), [(n, SCRIPT_ERR_NAMES[int(d)], SCRIPT_ERR_NAMES[int(h)]) for n, d, h in zip(names, dev, host) if d != h]
    assert len(b.arena) > 10000 and len(cases["10000-byte spk"][1]) == 10000
    assert got["244 items"][0] == "Ok" and got["245 items"][0] == "StackSizeExceeded" and got["243 + 3DUP"][0] == "StackSizeExceeded"
    assert got["201 hashes bare"][0] == "Ok" and got["202 hashes bare"][0] == "TooManyOperations"
    assert got["201 hashes in redeem"][0] == "Ok" and got["202 hashes in redeem"][0] == "TooManyOperations"
    assert got["201 IF deep"][0] == "ErrUnbalancedConditional" and got["10001-byte spk"][0] == "ScriptSize" and got["10000-byte spk"][0] == "Ok"
    assert got["checks: 9 multisig + 11 checksig"] == ("Ok", 9 * 20 + 11)  # 200 counted opcodes: the most checks one script reaches
    assert got["checks beyond sig_op_count"] == ("ExceededSigOpLimit", 50)


def test_slot_size(se):
    # stack 248 x 16 B + heap 203 x 32 B + condition stack: the per-input scratch the call budgets 64 MiB of
    assert se.hs_slot_bytes() == 248 * 16 + 203 * 32 + 204 + 4
