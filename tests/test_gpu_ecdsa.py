"""GPU parity: kgv_ecdsa_verify (through the C ABI) vs the CPU oracle on the same seeded inputs.
ECDSA verdicts are "parity unpinned" by reference vectors (SURVEY.md §8c): the oracle itself is
cross-checked against oracle/pyref.py and OpenSSL in tests/test_oracle_secp.py."""
import numpy as np
import pytest

from conftest import oracle_ecdsa_batch
from ladder_model import crafted_ecdsa_edge_cases
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu


def test_ecdsa_parity_mixed_batch(gpu_ctx, oracle):
    pk, msg, sig, kind = W.ecdsa_triples(12000, seed=2, n_keys=1024, n_nonces=1024, frac_bitflip=0.1, frac_adversarial=0.15)
    got = gpu_ctx.verify_ecdsa_batch(pk, msg, sig)
    exp = oracle_ecdsa_batch(oracle, pk, msg, sig)
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at {bad[:5]}: got {got[bad[:5]]} exp {exp[bad[:5]]} kind {kind[bad[:5]]}"
    assert (got[kind == 0] == 1).all()
    assert (got[kind != 0] != 1).all()
    assert set(np.unique(got)) == {0, 1, 2, 3}  # every verdict class is exercised


@pytest.mark.parametrize("n", [0, 1, 33, 129])
def test_ecdsa_ragged_sizes(gpu_ctx, oracle, n):
    pk, msg, sig, kind = W.ecdsa_triples(max(n, 1), seed=n + 11, n_keys=16, n_nonces=16, frac_bitflip=0.2, frac_adversarial=0.2)
    pk, msg, sig = pk[:n], msg[:n], sig[:n]
    got = gpu_ctx.verify_ecdsa_batch(pk, msg, sig, n=n)
    if n:
        assert (got == oracle_ecdsa_batch(oracle, pk, msg, sig)).all()


def test_ecdsa_crafted_edge_cases(gpu_ctx, oracle):
    """r + n < p wrap-around, the low-S boundary and foreign key tags: GPU == oracle == pyref == construction, and OpenSSL agrees where it has an opinion"""
    import pyref
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    cases = crafted_ecdsa_edge_cases()
    pk = np.frombuffer(b"".join(c[0] for c in cases), dtype=np.uint8).reshape(-1, 33).copy()
    msg = np.frombuffer(b"".join(c[1] for c in cases), dtype=np.uint8).reshape(-1, 32).copy()
    sig = np.frombuffer(b"".join(c[2] for c in cases), dtype=np.uint8).reshape(-1, 64).copy()
    exp = [c[3] for c in cases]
    assert gpu_ctx.verify_ecdsa_batch(pk, msg, sig).tolist() == exp
    assert oracle_ecdsa_batch(oracle, pk, msg, sig).tolist() == exp
    assert [pyref.ecdsa_verify(*(x.tobytes() for x in (pk[i], msg[i], sig[i]))) for i in range(len(cases))] == exp
    n_ossl = 0
    for (k, m, s, e, label) in cases:
        if k[0] not in (2, 3):
            continue
        pub = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP256K1(), k)
        try:
            pub.verify(utils.encode_dss_signature(int.from_bytes(s[:32], "big"), int.from_bytes(s[32:], "big")), m, ec.ECDSA(utils.Prehashed(hashes.SHA256())))
            ok = True
        except InvalidSignature:
            ok = False
        assert ok == (e == 1 or label == "s=high-boundary"), label  # OpenSSL accepts high S; libsecp256k1 (and this path) do not
        n_ossl += 1
    assert n_ossl >= 40 and sum(1 for c in cases if c[4] == "wrap") == 12


def test_ecdsa_gpu_verdicts_against_openssl(gpu_ctx):
    """a third, fully independent check of the GPU verdicts themselves (not via the oracle): OpenSSL (`cryptography`) with libsecp256k1's low-S rule
    added, over the whole 12 000-item mixed batch of the parity test"""
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec, utils
    N = W.N
    pk, msg, sig, kind = W.ecdsa_triples(12000, seed=2, n_keys=1024, n_nonces=1024, frac_bitflip=0.1, frac_adversarial=0.15)
    got = gpu_ctx.verify_ecdsa_batch(pk, msg, sig)
    checked = 0
    for i in range(len(pk)):
        r, s = int.from_bytes(sig[i, :32].tobytes(), "big"), int.from_bytes(sig[i, 32:].tobytes(), "big")
        try:
            pub = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP256K1(), pk[i].tobytes()) if pk[i, 0] in (2, 3) else None
        except ValueError:
            pub = None
        if pub is None:
            assert got[i] == 2, i
            continue
        if r >= N or s >= N:
            assert got[i] == 3, i
            continue
        if r == 0 or s == 0:
            assert got[i] == 0, i
            continue
        try:
            pub.verify(utils.encode_dss_signature(r, s), msg[i].tobytes(), ec.ECDSA(utils.Prehashed(hashes.SHA256())))
            ok = True
        except InvalidSignature:
            ok = False
        assert (got[i] == 1) == (ok and s <= N // 2), i
        checked += 1
    assert checked > 10000


def test_ecdsa_parity_100k_adversarial_heavy(gpu_ctx, oracle):
    """10^5 triples, 70 % of them corrupted or adversarially encoded (high S, r|s >= n, zero r|s, foreign tags, x >= p, off-curve keys, single-bit flips)"""
    pk, msg, sig, kind = W.ecdsa_triples(100_000, seed=41, n_keys=512, n_nonces=512, frac_bitflip=0.3, frac_adversarial=0.4)
    got = gpu_ctx.verify_ecdsa_batch(pk, msg, sig)
    exp = oracle_ecdsa_batch(oracle, pk, msg, sig)
    assert (got == exp).all() and (got[kind == 0] == 1).all() and not (got[kind != 0] == 1).any()
    assert min(np.bincount(got, minlength=4)) > 2000
