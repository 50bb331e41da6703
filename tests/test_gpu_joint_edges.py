"""The joint ladder's exceptional additions on the GPU (ecmult_joint, the comb form's ladder): signatures built by tests/joint_model.py
to reach its doubling fall-through and its cancellation to infinity at generator additions of both groups, at key additions after
them and at the combined parity fix, and Schnorr triples ending in R = infinity or meeting that fix.  They are verified inside a launch
that takes the comb form (kgv_debug_key_form confirms it), each in a thread whose other items are valid filler, and must equal the
oracle and the constructed verdicts; every filler verdict must equal that of the filler verified alone."""
import math

import numpy as np
import pytest

import joint_model as J
import ladder_model as L
from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

N_ITEMS, N_KEYS = 180_000, 2048  # several items per thread of an H100's resident grid, about 88 uses per key: the comb form


def _verify(gpu_ctx, kind, pk, msg, sig):
    import torch
    bufs = [torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda() for a in (pk, msg, sig)]
    st = torch.empty(len(pk), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    (gpu_ctx.verify_ecdsa_batch if kind == "ecdsa" else gpu_ctx.verify_schnorr_batch)(*bufs, n=len(pk), status=st)
    info = gpu_ctx.debug_key_form(ecdsa=kind == "ecdsa")
    torch.cuda.synchronize()
    return st.cpu().numpy(), info


def _placement(n, T, fkind, count):
    """`count` item positions in distinct threads whose other items are valid filler"""
    step = 97
    while math.gcd(step, T) != 1:
        step += 2
    pos = []
    for k in range(T):
        t = (5 + k * step) % T
        items = list(range(t, n, T))
        j = len(pos) % len(items)
        if all(fkind[i] == 0 for i in items if i != items[j]):
            pos.append(items[j])
            if len(pos) == count:
                return np.array(pos)
    raise AssertionError("not enough threads with valid filler")


@pytest.mark.parametrize("kind", ["schnorr", "ecdsa"])
def test_joint_ladder_edges_in_the_comb_form(gpu_ctx, oracle, kind):
    cs = J.ecdsa_joint_cases(oracle) if kind == "ecdsa" else J.schnorr_infinity_and_fix_cases(oracle)
    cpk, cmsg, csig = L.arrays(cs)
    cexp = np.array([c["exp"] for c in cs], dtype=np.uint8)
    ora = (oracle_ecdsa_batch if kind == "ecdsa" else oracle_schnorr_batch)(oracle, cpk, cmsg, csig)
    assert (ora == cexp).all(), [cs[i]["label"] for i in np.nonzero(ora != cexp)[0][:5]]
    if kind == "ecdsa":
        assert {c["sigma"] for c in cs} == {1, -1} and any(c["exp"] == 1 for c in cs)
    keys, nonces = W.ScalarPointPool(N_KEYS, 71, b"keys"), W.ScalarPointPool(1024, 71, b"nonces")
    gen = W.ecdsa_triples if kind == "ecdsa" else W.schnorr_triples
    fpk, fmsg, fsig, fkind = gen(N_ITEMS, seed=72, frac_bitflip=0.01, frac_adversarial=0.01, pools=(keys, nonces))
    alone, info = _verify(gpu_ctx, kind, fpk, fmsg, fsig)
    assert info["form"] == "comb", info
    assert (alone[fkind == 0] == 1).all() and not (alone[fkind != 0] == 1).any()
    pos = _placement(N_ITEMS, info["threads"], fkind, len(cexp))
    pk, msg, sig, exp = fpk.copy(), fmsg.copy(), fsig.copy(), alone.copy()
    pk[pos], msg[pos], sig[pos], exp[pos] = cpk, cmsg, csig, cexp
    got, info = _verify(gpu_ctx, kind, pk, msg, sig)
    assert info["form"] == "comb", info
    bad = np.nonzero(got[pos] != cexp)[0]
    assert len(bad) == 0, [(cs[i]["label"], int(got[pos][i]), int(cexp[i])) for i in bad[:8]]
    bad = np.nonzero(got != exp)[0]
    assert len(bad) == 0, f"items {bad[:8]}: got {got[bad[:8]]} exp {exp[bad[:8]]}"
