"""Comb key records (key_comb_build / ecmult_comb, DESIGN.md §4 K1): a launch whose keys are used at least KGV_COMB_USES (8) times on
average prepares each key as a four-tooth comb and runs the 32-doubling ladder.  Every verdict is compared with the CPU oracle, on
launches that take the comb form and on launches just outside it."""
import numpy as np
import pytest

from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

P = 2**256 - 2**32 - 977
COMB_USES = 8


def _tiled(base, exp, n):
    pk, msg, sig, kind = W.tile_triples(*base, n)
    return pk, msg, sig, kind, np.tile(exp, (n + len(exp) - 1) // len(exp))[:n]


def _check(got, exp):
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at {bad[:5]}: got {got[bad[:5]]} exp {exp[bad[:5]]}"


@pytest.mark.parametrize("n_keys", [1, 1024])
def test_comb_keys_with_corrupted_items(gpu_ctx, oracle, n_keys):
    base = W.schnorr_triples(20000, seed=31 + n_keys, n_keys=n_keys, n_nonces=2048, frac_bitflip=0.05, frac_adversarial=0.05)
    exp = oracle_schnorr_batch(oracle, *base[:3])
    pk, msg, sig, kind, exp = _tiled(base, exp, 210_000)
    assert COMB_USES * len(np.unique(pk, axis=0)) <= len(pk)
    got = gpu_ctx.verify_schnorr_batch(pk, msg, sig)
    _check(got, exp)
    assert (got[kind == 0] == 1).all() and not (got[kind != 0] == 1).any()


def test_comb_repeated_bad_keys(gpu_ctx, oracle):
    pk, msg, sig, kind = W.tile_triples(*W.schnorr_triples(3000, seed=33, n_keys=8, n_nonces=64, frac_bitflip=0.0, frac_adversarial=0.0), 120000)
    rng = np.random.default_rng(33)
    pk[0:10000] = np.frombuffer((P + 5).to_bytes(32, "big"), dtype=np.uint8)
    pk[10000:20000] = np.frombuffer(W._non_residue_x(rng).to_bytes(32, "big"), dtype=np.uint8)
    got = gpu_ctx.verify_schnorr_batch(pk, msg, sig)
    _check(got, oracle_schnorr_batch(oracle, pk, msg, sig))
    assert (got[:20000] == 2).all() and (got[20000:] == 1).all()


def test_comb_ecdsa_tags(gpu_ctx, oracle):
    base = W.ecdsa_triples(6000, seed=34, n_keys=64, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05)
    pk, msg, sig, kind = W.tile_triples(*base, 100000)
    flip = pk.copy()
    ok = (flip[:, 0] == 2) | (flip[:, 0] == 3)
    flip[ok, 0] ^= 1  # the same x under the other tag: a second key
    both = lambda a, b: np.ascontiguousarray(np.concatenate([a, b]))
    pk2, msg2, sig2 = both(pk, flip), both(msg, msg), both(sig, sig)
    assert COMB_USES * len(np.unique(pk2, axis=0)) <= len(pk2)
    got = gpu_ctx.verify_ecdsa_batch(pk2, msg2, sig2)
    _check(got, oracle_ecdsa_batch(oracle, pk2, msg2, sig2))
    assert (got[:100000][kind == 0] == 1).all() and not (got[100000:] == 1).any()


def test_comb_unaligned_device_buffers(gpu_ctx, oracle):
    import torch
    base = W.schnorr_triples(5000, seed=35, n_keys=32, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05)
    pk, msg, sig, kind, exp = _tiled(base, oracle_schnorr_batch(oracle, *base[:3]), 100000)
    for off in (1, 16):
        bufs = []
        for a in (pk, msg, sig):
            t = torch.zeros(a.nbytes + off, dtype=torch.uint8, device="cuda")
            t[off:] = torch.from_numpy(a.reshape(-1)).cuda()
            bufs.append(t[off:])
        st = torch.empty(100000, dtype=torch.uint8, device="cuda")
        gpu_ctx.verify_schnorr_batch(*bufs, n=100000, status=st)
        torch.cuda.synchronize()
        _check(st.cpu().numpy(), exp)


@pytest.mark.parametrize("extra", [0, 1])
def test_key_count_at_the_comb_threshold(gpu_ctx, oracle, extra):
    # d distinct keys over n = 8d items takes the comb form; over 8d - 1 items the plain records
    base = W.schnorr_triples(40000, seed=36, n_keys=8000, n_nonces=2048, frac_bitflip=0.02, frac_adversarial=0.02)
    d = len(np.unique(base[0], axis=0))
    n = COMB_USES * d - extra
    assert n >= len(base[0])
    pk, msg, sig, kind, exp = _tiled(base, oracle_schnorr_batch(oracle, *base[:3]), n)
    assert len(np.unique(pk, axis=0)) == d
    _check(gpu_ctx.verify_schnorr_batch(pk, msg, sig), exp)


def test_comb_indexed_launches_through_the_signature_cache(gpu_ctx, oracle):
    """The INDEXED kernels on the signature-cache misses of a validation call over few keys (the comb form), against the oracle."""
    import oracle_tx
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import Params, SigCache, TransactionValidator
    fk, fe, txs = simgen.funded_window(70000, n_keys=16, n_nonces=64, mix=(0.5, 0.3, 0.1, 0.1))
    ents, k = [], 0
    for t in txs:
        ents.append(fe[k:k + len(t["inputs"])])
        k += len(t["inputs"])
    rng = np.random.default_rng(37)
    for i in rng.choice(len(txs), size=60, replace=False):
        ss = bytearray(txs[i]["inputs"][0]["sigscript"])
        ss[5 + int(rng.integers(0, 50))] ^= 1 << int(rng.integers(0, 8))
        txs[i]["inputs"][0]["sigscript"] = bytes(ss)
    b = build_batch(txs, ents)
    tv = TransactionValidator(gpu_ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    exp = [oracle_tx.validate_populated(oracle, b, i, 10, 0, op) for i in range(len(txs))]
    sc = SigCache(gpu_ctx, 1 << 14)
    sc.attach()
    try:
        r = tv.validate_populated_transactions(b, 10)
        for i in range(len(txs)):
            assert int(r["status"][i]) == int(exp[i]["status"]) and int(r["fee"][i]) == int(exp[i]["fee"]), (i, r[i], exp[i])
    finally:
        sc.close()
