"""Pins the C oracle's curve arithmetic: BIP-340 official vector, agreement with the independent big-int
twin (oracle/pyref.py) and with OpenSSL (`cryptography`) on random + adversarial inputs.
ECDSA verdicts / Schnorr edge encodings have no stored vector in the reference ("parity unpinned",
SURVEY.md §8c) — this three-way agreement is the mitigation the survey prescribes."""
import ctypes
import random

import numpy as np
import pytest

import pyref
from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W


def test_bip340_vector0(oracle):
    sk = bytes.fromhex("0000000000000000000000000000000000000000000000000000000000000003")
    pk = bytes.fromhex("F9308A019258C31049344F85F89D5229B531C845836F99B08601F113BCE036F9")
    sig = bytes.fromhex("E907831F80848D1069A5371B402410364BDF1C5F8307B0084C55F1CE2DCA8215"
                        "25F66A4A85EA8B71E482A74F382D2CE5EBEEE8FDB2172F477DF4900D310536C0")
    out = ctypes.create_string_buffer(64)
    assert oracle.ok_schnorr_sign(sk, bytes(32), out) == 1 and out.raw == sig
    assert pyref.schnorr_sign(sk, bytes(32)) == sig
    assert oracle.ok_schnorr_verify(pk, bytes(32), sig) == 1


def test_field_and_scalar_mul_vs_bigint(oracle):
    rnd = random.Random(1)
    o = ctypes.create_string_buffer(32)
    for _ in range(2000):
        a, b = rnd.randrange(2**256), rnd.randrange(2**256)
        oracle.ok_fe_mul_bytes(a.to_bytes(32, "big"), b.to_bytes(32, "big"), o)
        assert int.from_bytes(o.raw, "big") == a * b % pyref.P
        oracle.ok_sc_mul_bytes(a.to_bytes(32, "big"), b.to_bytes(32, "big"), o)
        assert int.from_bytes(o.raw, "big") == a * b % pyref.N


def test_schnorr_oracle_vs_pyref():
    import conftest
    pk, msg, sig, kind = W.schnorr_triples(240, seed=31, n_keys=8, n_nonces=8, frac_bitflip=0.25, frac_adversarial=0.4)
    lib = ctypes.CDLL(conftest.os.path.join(conftest.ROOT, "oracle", "libkaspa_oracle.so"))
    lib.ok_secp_init()
    st = oracle_schnorr_batch(lib, pk, msg, sig, threads=1)
    for i in range(len(pk)):
        assert pyref.schnorr_verify(pk[i].tobytes(), msg[i].tobytes(), sig[i].tobytes()) == st[i], (i, kind[i])
    assert set(st) == {0, 1, 2}


def test_ecdsa_oracle_vs_pyref_and_openssl(oracle):
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    pk, msg, sig, kind = W.ecdsa_triples(600, seed=32, n_keys=16, n_nonces=16, frac_bitflip=0.2, frac_adversarial=0.3)
    st = oracle_ecdsa_batch(oracle, pk, msg, sig, threads=1)
    assert set(st) == {0, 1, 2, 3}
    checked = 0
    for i in range(len(pk)):
        if i % 4 == 0:
            assert pyref.ecdsa_verify(pk[i].tobytes(), msg[i].tobytes(), sig[i].tobytes()) == st[i], (i, kind[i])
        if st[i] in (2, 3):
            continue
        r, s = int.from_bytes(sig[i, :32].tobytes(), "big"), int.from_bytes(sig[i, 32:].tobytes(), "big")
        if r == 0 or s == 0:
            continue
        pub = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP256K1(), pk[i].tobytes())
        try:
            pub.verify(utils.encode_dss_signature(r, s), msg[i].tobytes(), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
            ossl = True
        except InvalidSignature:
            ossl = False
        # libsecp256k1 additionally requires low S (OpenSSL does not)
        assert (st[i] == 1) == (ossl and s <= pyref.N // 2), i
        checked += 1
    assert checked > 300


def test_sign_roundtrip_matches_pyref(oracle):
    rnd = random.Random(5)
    for _ in range(10):
        sk, m = bytes(rnd.getrandbits(8) for _ in range(32)), bytes(rnd.getrandbits(8) for _ in range(32))
        pk, sig = ctypes.create_string_buffer(32), ctypes.create_string_buffer(64)
        assert oracle.ok_schnorr_pubkey(sk, pk) and oracle.ok_schnorr_sign(sk, m, sig)
        assert pk.raw == pyref.schnorr_pubkey(sk) and sig.raw == pyref.schnorr_sign(sk, m)
        assert oracle.ok_schnorr_verify(pk.raw, m, sig.raw) == 1
        pk33 = ctypes.create_string_buffer(33)
        assert oracle.ok_ecdsa_pubkey(sk, pk33) and oracle.ok_ecdsa_sign(sk, m, sig)
        assert pk33.raw == pyref.ecdsa_pubkey(sk)
        assert oracle.ok_ecdsa_verify(pk33.raw, m, sig.raw) == 1 == pyref.ecdsa_verify(pk33.raw, m, sig.raw)


def test_bip340_test_vectors(oracle):
    """rows 0-14 of BIP-340's own test-vectors.csv (tests/golden/bip340_vectors.csv): signing KATs, a low-r signature, and every
    malformed-encoding case the BIP lists (off-curve key, odd-y R, negated message / s, R at infinity, r not on the curve, r = p,
    s = n, key >= p) through the C oracle and the Python twin"""
    import pyref
    from conftest import oracle_schnorr_batch
    from golden_util import bip340_vectors
    pk, msg, sig, exp, comments = bip340_vectors()
    assert len(exp) == 15 and exp.count(1) == 5 and exp.count(2) == 2
    got = oracle_schnorr_batch(oracle, pk, msg, sig, threads=2)
    assert got.tolist() == exp, [(i, c) for i, (g, e, c) in enumerate(zip(got, exp, comments)) if g != e]
    assert [pyref.schnorr_verify(pk[i].tobytes(), msg[i].tobytes(), sig[i].tobytes()) for i in range(15)] == exp


def _batch(fn, pk, msg, sig, threads=4):
    import numpy as np
    st = np.zeros(len(pk), dtype=np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    fn(vp(pk), vp(msg), vp(sig), ctypes.c_size_t(len(pk)), vp(st), threads)
    return st


def test_fast_cpu_port_equals_the_plain_checker(oracle):
    """oracle/ok_secp_fast.c (GLV + wNAF + effective-affine tables: the port the CPU baselines time) must return the plain checker's verdicts
    bit for bit: mixed Schnorr and ECDSA batches with every adversarial class, the BIP-340 vectors, the crafted ECDSA edge cases (r + n < p wrap,
    low-S boundary, foreign key tags), and scalars that stress the GLV split (tiny, huge, near n/2, near lambda multiples)"""
    import numpy as np
    from golden_util import bip340_vectors
    pk, msg, sig, kind = W.schnorr_triples(6000, seed=13, n_keys=512, n_nonces=512, frac_bitflip=0.15, frac_adversarial=0.15)
    a, b = _batch(oracle.ok_schnorr_verify_batch, pk, msg, sig), _batch(oracle.ok_schnorr_verify_batch_fast, pk, msg, sig)
    assert (a == b).all() and set(a) == {0, 1, 2}
    pk, msg, sig, kind = W.ecdsa_triples(6000, seed=14, n_keys=512, n_nonces=512, frac_bitflip=0.15, frac_adversarial=0.2)
    a, b = _batch(oracle.ok_ecdsa_verify_batch, pk, msg, sig), _batch(oracle.ok_ecdsa_verify_batch_fast, pk, msg, sig)
    assert (a == b).all() and set(a) == {0, 1, 2, 3}
    bpk, bmsg, bsig, exp, _ = bip340_vectors()
    assert _batch(oracle.ok_schnorr_verify_batch_fast, bpk, bmsg, bsig).tolist() == exp
    from ladder_model import crafted_ecdsa_edge_cases
    cases = crafted_ecdsa_edge_cases()
    cpk = np.frombuffer(b"".join(c[0] for c in cases), dtype=np.uint8).reshape(-1, 33).copy()
    cmsg = np.frombuffer(b"".join(c[1] for c in cases), dtype=np.uint8).reshape(-1, 32).copy()
    csig = np.frombuffer(b"".join(c[2] for c in cases), dtype=np.uint8).reshape(-1, 64).copy()
    assert _batch(oracle.ok_ecdsa_verify_batch_fast, cpk, cmsg, csig).tolist() == [c[3] for c in cases]
    # ECDSA with hand-picked u2 = r/s values that stress the endomorphism split: Q = d*G, choose s so that u2 hits the target
    N, G = pyref.N, pyref.G
    lam = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
    rnd = random.Random(8)
    rows = []
    for target in [1, 2, N - 1, N - 2, (N - 1) // 2, (N + 1) // 2, lam, N - lam, (lam * 3) % N, 2**128, 2**128 - 1, 2**129 + 5, (lam + 1) % N, (lam * lam) % N]:
        d, k = rnd.randrange(1, N), rnd.randrange(1, N)
        r = pyref.pt_mul(k, G)[0] % N
        s = r * pow(target, -1, N) % N           # u2 = r / s = target
        m = (s * k - r * d) % N                  # makes the signature valid
        if s > N // 2:                            # keep low S (negating s negates u1, u2: still exercises |u2| = target)
            s, m = N - s, m                       # now invalid for this message; both ports must still agree
        Q = pyref.pt_mul(d, G)
        rows.append((bytes([2 + (Q[1] & 1)]) + Q[0].to_bytes(32, "big"), m.to_bytes(32, "big"), r.to_bytes(32, "big") + s.to_bytes(32, "big")))
    gpk = np.frombuffer(b"".join(x[0] for x in rows), dtype=np.uint8).reshape(-1, 33).copy()
    gmsg = np.frombuffer(b"".join(x[1] for x in rows), dtype=np.uint8).reshape(-1, 32).copy()
    gsig = np.frombuffer(b"".join(x[2] for x in rows), dtype=np.uint8).reshape(-1, 64).copy()
    a, b = _batch(oracle.ok_ecdsa_verify_batch, gpk, gmsg, gsig), _batch(oracle.ok_ecdsa_verify_batch_fast, gpk, gmsg, gsig)
    assert (a == b).all() and 1 in a
