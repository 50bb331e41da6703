"""The per-launch key cache of the verify kernels (k_key_dedup / k_key_prepare): in a launch whose keys repeat, every distinct public
key is prepared once and its record replaces the per-signature key work.  Verdicts are checked against the CPU oracle on batches that
take the record path and the inline path, with good keys, unparseable keys, near-identical keys and more keys than records.  The
cache runs in launches of more items than the device has resident threads (50 688 on an H100), so every batch here is larger."""
import numpy as np
import pytest

from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

P = 2**256 - 2**32 - 977


def _check_schnorr(ctx, oracle, pk, msg, sig, exp=None):
    got = ctx.verify_schnorr_batch(pk, msg, sig)
    if exp is None:
        exp = oracle_schnorr_batch(oracle, pk, msg, sig)
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at {bad[:5]}: got {got[bad[:5]]} exp {exp[bad[:5]]}"
    return got


def _check_ecdsa(ctx, oracle, pk, msg, sig):
    got = ctx.verify_ecdsa_batch(pk, msg, sig)
    exp = oracle_ecdsa_batch(oracle, pk, msg, sig)
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at {bad[:5]}: got {got[bad[:5]]} exp {exp[bad[:5]]}"
    return got


def test_one_key_100k_items(gpu_ctx, oracle):
    pk, msg, sig, kind = W.schnorr_triples(2000, seed=11, n_keys=1, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05)
    exp = oracle_schnorr_batch(oracle, pk, msg, sig)
    pk, msg, sig, kind = W.tile_triples(pk, msg, sig, kind, 100_000)
    got = _check_schnorr(gpu_ctx, oracle, pk, msg, sig, np.tile(exp, 50)[:100_000])
    assert (got[kind == 0] == 1).all()


@pytest.mark.parametrize("n_keys", [64, 20000, 1 << 30])
def test_reuse_distinct_and_mixed(gpu_ctx, oracle, n_keys):
    # 64 keys: every key repeated; n_keys >= n: keys mostly used once (no records); 20000 keys over 60000 items: singletons beside
    # repeated keys, all with records
    pk, msg, sig, kind = W.schnorr_triples(60000, seed=12, n_keys=n_keys, n_nonces=1024, frac_bitflip=0.05, frac_adversarial=0.05)
    got = _check_schnorr(gpu_ctx, oracle, pk, msg, sig)
    assert (got[kind == 0] == 1).all()


def test_repeated_bad_keys(gpu_ctx, oracle):
    pk, msg, sig, kind = W.tile_triples(*W.schnorr_triples(3000, seed=13, n_keys=8, n_nonces=64, frac_bitflip=0.0, frac_adversarial=0.0), 60000)
    rng = np.random.default_rng(13)
    ge_p = (P + 5).to_bytes(32, "big")
    off_curve = W._non_residue_x(rng).to_bytes(32, "big")
    pk[0:10000] = np.frombuffer(ge_p, dtype=np.uint8)
    pk[10000:20000] = np.frombuffer(off_curve, dtype=np.uint8)
    got = _check_schnorr(gpu_ctx, oracle, pk, msg, sig)
    assert (got[:20000] == 2).all() and (got[20000:] == 1).all()


def test_keys_differing_in_one_byte(gpu_ctx, oracle):
    # every key appears unchanged and with one byte changed (each byte position, several flips), all repeated: the full-key compare
    # must keep them apart however their fingerprints and slots fall
    pk, msg, sig, kind = W.tile_triples(*W.schnorr_triples(4096, seed=14, n_keys=4, n_nonces=256, frac_bitflip=0.0, frac_adversarial=0.0), 65536)
    for i in range(0, 65536, 2):
        pk[i, (i // 2) % 32] ^= 1 << ((i // 64) % 8)
    got = _check_schnorr(gpu_ctx, oracle, pk, msg, sig)
    assert (got[1::2] == 1).all() and (got[0::2] != 1).all()


def test_more_repeated_keys_than_records(gpu_ctx, oracle):
    # 260000 items over 260000 keys, then the same items again: about 164000 distinct keys, above the 2^17 records of one launch,
    # so the launch makes none and every item verifies on the inline path
    pk, msg, sig, kind = W.schnorr_triples(260000, seed=15, n_keys=260000, n_nonces=4096, frac_bitflip=0.01, frac_adversarial=0.01)
    exp = oracle_schnorr_batch(oracle, pk, msg, sig)
    assert len(np.unique(pk, axis=0)) > (1 << 17)
    cat = lambda a: np.ascontiguousarray(np.concatenate([a, a]))
    got = _check_schnorr(gpu_ctx, oracle, cat(pk), cat(msg), cat(sig), np.concatenate([exp, exp]))
    assert (got[:260000][kind == 0] == 1).all()


def test_unaligned_device_buffers(gpu_ctx, oracle):
    import torch
    pk, msg, sig, kind = W.schnorr_triples(5000, seed=16, n_keys=32, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05)
    exp = np.tile(oracle_schnorr_batch(oracle, pk, msg, sig), 12)
    pk, msg, sig, kind = W.tile_triples(pk, msg, sig, kind, 60000)
    for off in (1, 3, 16):
        bufs = []
        for a in (pk, msg, sig):
            t = torch.zeros(a.nbytes + off, dtype=torch.uint8, device="cuda")
            t[off:] = torch.from_numpy(a.reshape(-1)).cuda()
            bufs.append(t[off:])
        st = torch.empty(60000, dtype=torch.uint8, device="cuda")
        gpu_ctx.verify_schnorr_batch(*bufs, n=60000, status=st)
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == exp).all(), off


def test_ecdsa_reuse_and_tags(gpu_ctx, oracle):
    pk, msg, sig, kind = W.tile_triples(*W.ecdsa_triples(6000, seed=17, n_keys=32, n_nonces=256, frac_bitflip=0.05, frac_adversarial=0.05), 60000)
    _check_ecdsa(gpu_ctx, oracle, pk, msg, sig)
    # the same x under tag 02 and 03 in one batch: two different keys, each repeated
    flip = pk.copy()
    ok = (flip[:, 0] == 2) | (flip[:, 0] == 3)
    flip[ok, 0] ^= 1
    both = lambda a, b: np.ascontiguousarray(np.concatenate([a, b]))
    got = _check_ecdsa(gpu_ctx, oracle, both(pk, flip), both(msg, msg), both(sig, sig))
    assert (got[:60000][kind == 0] == 1).all() and not (got[60000:] == 1).any()
    # a bad tag and an off-curve x, repeated
    bad = pk.copy()
    bad[:5000, 0] = 4
    bad[5000:10000, 1:] = np.frombuffer(W._non_residue_x(np.random.default_rng(17)).to_bytes(32, "big"), dtype=np.uint8)
    got = _check_ecdsa(gpu_ctx, oracle, bad, msg, sig)
    assert (got[:10000] == 2).all()


def test_indexed_launches_through_the_signature_cache(gpu_ctx, oracle):
    """Validation with the signature cache attached verifies only the cache misses (the INDEXED kernels, count on the device):
    few keys, Schnorr and ECDSA spends (more than 50 688 signature checks of each kind), some corrupted signatures and unparseable keys,
    against the oracle's validator."""
    import oracle_tx
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.txbatch import build_batch
    from rusty_kaspa_b200.validator import Params, SigCache, TransactionValidator
    fk, fe, txs = simgen.funded_window(60000, n_keys=8, n_nonces=64, mix=(0.4, 0.4, 0.1, 0.1))
    ents, k = [], 0
    for t in txs:
        ents.append(fe[k:k + len(t["inputs"])])
        k += len(t["inputs"])
    rng = np.random.default_rng(18)
    for i in rng.choice(len(txs), size=60, replace=False):
        ss = bytearray(txs[i]["inputs"][0]["sigscript"])
        ss[5 + int(rng.integers(0, 50))] ^= 1 << int(rng.integers(0, 8))
        txs[i]["inputs"][0]["sigscript"] = bytes(ss)
    for i in rng.choice(len(txs), size=30, replace=False):
        e = ents[i][0]
        if len(e["script"]) == 34:
            ents[i][0] = dict(e, script=bytes([0x20]) + W._non_residue_x(rng).to_bytes(32, "big") + bytes([0xAC]))
    b = build_batch(txs, ents)
    tv = TransactionValidator(gpu_ctx, Params(storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER))
    op = oracle_tx.params(coinbase_maturity=100, storage_mass_parameter=simgen.DEFAULT_STORAGE_MASS_PARAMETER)
    exp = [oracle_tx.validate_populated(oracle, b, i, 10, 0, op) for i in range(len(txs))]
    sc = SigCache(gpu_ctx, 1 << 14)
    sc.attach()
    try:
        for _ in range(2):  # all misses, then mostly hits
            r = tv.validate_populated_transactions(b, 10)
            for i in range(len(txs)):
                assert int(r["status"][i]) == int(exp[i]["status"]) and int(r["fee"][i]) == int(exp[i]["fee"]), (i, r[i], exp[i])
        assert sc.counters()["hits"] > 0
    finally:
        sc.close()
