"""The verify ladders' exceptional additions on the GPU, in every key form: signatures built by tests/ladder_model.py to reach the
doubling fall-through, the cancellation to infinity and the addition onto infinity in the middle of a ladder, verified in launches
that take the inline form (one item per thread, and several items per thread with too many keys for records), the plain key records
and the comb records.  kgv_debug_key_form confirms the form of every launch.

Each launch holds the crafted sets of both ladders (the other ladder's set runs as ordinary items), filler, and threads whose items
are all R = infinity or all parse failures (the phase-2 pass of such a thread has nothing to invert).  Crafted items sit in threads
whose other items (i + j*T for the grid's T threads share one inversion) are valid filler, and move over lane positions between
launches.  Every crafted verdict must equal the plain oracle and the constructed one; every filler verdict must equal the verdict of
the same filler verified alone."""
import math

import numpy as np
import pytest

import ladder_model as L
from conftest import oracle_ecdsa_batch, oracle_schnorr_batch
from rusty_kaspa_b200 import workload as W

pytestmark = pytest.mark.gpu

N_LARGE = 180_000  # more than three items per thread of an H100's resident grid (50 688 threads), fewer than four
N_SMALL = 8192
# form -> (items, distinct filler keys)
FORMS = {"no-cache": (N_SMALL, 256), "inline": (N_LARGE, N_LARGE), "plain": (N_LARGE, 40_000), "comb": (N_LARGE, 2048)}


@pytest.fixture(scope="module")
def crafted(oracle):
    out = {}
    for kind, cs in (("ecdsa", list(L.ecdsa_ladder_cases(oracle)) + L.ecdsa_edge_cases()),
                     ("schnorr", list(L.schnorr_ladder_cases(oracle)) + L.bip340_cases())):
        pk, msg, sig = L.arrays(cs)
        exp = np.array([c["exp"] for c in cs], dtype=np.uint8)
        ora = (oracle_ecdsa_batch if kind == "ecdsa" else oracle_schnorr_batch)(oracle, pk, msg, sig)
        assert (ora == exp).all(), [cs[i]["label"] for i in np.nonzero(ora != exp)[0][:5]]
        out[kind] = (pk, msg, sig, exp)
    return out


@pytest.fixture(scope="module")
def pools():
    return W.ScalarPointPool(N_LARGE, 61, b"keys"), W.ScalarPointPool(1024, 61, b"nonces")


def _filler(kind, form, pools):
    n, n_keys = FORMS[form]
    keys = pools[0] if n_keys == N_LARGE else W.ScalarPointPool(n_keys, 62, b"keys")
    gen = W.ecdsa_triples if kind == "ecdsa" else W.schnorr_triples
    return gen(n, seed=63, frac_bitflip=0.01, frac_adversarial=0.01, pools=(keys, pools[1])), keys


def _special(kind, keys, rng, what):
    """one item of a thread whose items all fail: R = infinity (what == "inf") or a parse failure (what == "parse")"""
    i = int(rng.integers(0, keys.count))
    d, px = keys.scalars[i], keys.xs[i]
    r = int(rng.integers(1, 2**62)) * 0x1000003D1 % L.N or 1
    m = rng.bytes(32)
    if kind == "schnorr":
        if what == "parse":
            return (L.P + 5).to_bytes(32, "big"), m, rng.bytes(64), 2
        rb = r.to_bytes(32, "big")
        return px, m, rb + (L._challenge(rb, px, m) * d % L.N).to_bytes(32, "big"), 0
    if what == "parse":
        return b"\x02" + px, m, (L.N + r).to_bytes(32, "big") + r.to_bytes(32, "big"), 3
    s = int(rng.integers(1, 2**62))
    return b"\x02" + px, (-r * d % L.N).to_bytes(32, "big"), r.to_bytes(32, "big") + s.to_bytes(32, "big"), 0  # u1 = -u2*d


def _verify(gpu_ctx, kind, pk, msg, sig, offset=0):
    """one launch on device buffers (offset > 0: misaligned by that many bytes); returns (verdicts, key form info)"""
    import torch
    bufs = []
    for a in (pk, msg, sig):
        t = torch.zeros(a.nbytes + offset, dtype=torch.uint8, device="cuda")
        t[offset:] = torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda()
        bufs.append(t[offset:])
    st = torch.empty(len(pk), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    (gpu_ctx.verify_ecdsa_batch if kind == "ecdsa" else gpu_ctx.verify_schnorr_batch)(*bufs, n=len(pk), status=st)
    info = gpu_ctx.debug_key_form(ecdsa=kind == "ecdsa")
    torch.cuda.synchronize()
    return st.cpu().numpy(), info


def _placement(n, T, fkind, count, shift, reserved):
    """`count` item positions in distinct threads whose other items are valid filler, starting at a lane that moves with `shift`"""
    step = 97
    while math.gcd(step, T) != 1:
        step += 2
    pos, tau = [], (shift * 13) % T
    for k in range(T):
        t = (tau + k * step) % T
        items = list(range(t, n, T))
        if t in reserved or not items:
            continue
        j = (len(pos) + shift) % len(items)
        if all(fkind[i] == 0 for i in items if i != items[j]):
            pos.append(items[j])
            if len(pos) == count:
                return np.array(pos)
    raise AssertionError("not enough threads with valid filler")


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("kind", ["schnorr", "ecdsa"])
def test_ladder_edges_in_every_key_form(gpu_ctx, crafted, pools, kind, form):
    (fpk, fmsg, fsig, fkind), keys = _filler(kind, form, pools)
    n = len(fpk)
    alone, info = _verify(gpu_ctx, kind, fpk, fmsg, fsig)
    assert info["n_items"] == n
    assert (alone[fkind == 0] == 1).all() and not (alone[fkind != 0] == 1).any()
    T = info["threads"]
    assert (n <= T) == (form == "no-cache")
    cpk, cmsg, csig, cexp = crafted[kind]
    rng = np.random.default_rng(64)
    for shift in range(3):
        pk, msg, sig, exp = fpk.copy(), fmsg.copy(), fsig.copy(), alone.copy()
        # threads whose four items all fail (need n > 3T)
        reserved = set()
        if form != "no-cache":
            assert n > 3 * T
            for t, what in ((shift * 32 + 1, "inf"), (shift * 32 + 2, "inf"), (shift * 32 + 33, "parse"), (shift * 32 + 70, "parse")):
                reserved.add(t)
                for i in range(t, n, T):
                    a, b, c, e = _special(kind, keys, rng, what)
                    pk[i], msg[i], sig[i], exp[i] = np.frombuffer(a, np.uint8), np.frombuffer(b, np.uint8), np.frombuffer(c, np.uint8), e
        pos = _placement(n, T, fkind, len(cexp), shift, reserved)
        pk[pos], msg[pos], sig[pos], exp[pos] = cpk, cmsg, csig, cexp
        got, info = _verify(gpu_ctx, kind, pk, msg, sig, offset=1 if shift == 2 else 0)
        assert info["form"] == form and info["n_items"] == n and info["threads"] == T, info
        bad = np.nonzero(got[pos] != cexp)[0]
        assert len(bad) == 0, f"{form} shift {shift}: crafted items {bad[:8]}: got {got[pos][bad[:8]]} exp {cexp[bad[:8]]}"
        bad = np.nonzero(got != exp)[0]
        assert len(bad) == 0, f"{form} shift {shift}: items {bad[:8]}: got {got[bad[:8]]} exp {exp[bad[:8]]}"


def test_model_split_against_the_device(gpu_ctx):
    """glv_split on the device (debug_selftest op 11) == the model's, over 10 000+ scalars incl. the edges"""
    import random
    rnd = random.Random(65)
    N, lam = L.N, L.LAMBDA
    ks = [0, 1, 2, N - 1, N - 2, 2**128 - 1, 2**128, 2**128 + 1, lam, N - lam, (2**128 * lam) % N, (2**128 - 1) * lam % N,
          (2**128 + 1) * lam % N, (N - 1) // 2, (N + 1) // 2, (-(1 + lam)) % N]
    ks += [rnd.randrange(N) for _ in range(10000)] + [rnd.randrange(2**130) for _ in range(500)]
    out = gpu_ctx.debug_selftest(11, ks, [0] * len(ks))
    for k, o in zip(ks, out):
        k1, n1, k2, n2 = L.glv_split(k)
        w = [(o >> (32 * i)) & 0xFFFFFFFF for i in range(16)]
        got = (sum(w[i] << (32 * i) for i in range(5)), bool(w[5]), sum(w[8 + i] << (32 * i) for i in range(5)), bool(w[13]))
        assert got == (k1, n1, k2, n2), hex(k)


def test_schnorr_trace_against_the_model(gpu_ctx, oracle):
    """debug_schnorr_trace (the device's ecmult_double, one thread) against the model for every crafted Schnorr case"""
    for c in L.schnorr_ladder_cases(oracle):
        assert L.check_schnorr_trace(gpu_ctx.debug_schnorr_trace, c) == 0, c["label"]
