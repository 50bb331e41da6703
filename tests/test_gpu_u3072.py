"""GPU: the MuHash field arithmetic (kgv_u3072.cuh, kgv_muhash.cu) on chosen operands, exactly against Python integers.

Hashed elements are uniformly random 3072-bit numbers and never reach the multipliers' rare paths (a third fold round, block
carries into all-ones blocks, values in [p, 2^3072)); here both tree-level kernels get the operands of tests/u3072_model.py
through kgv_debug_u3072_level, and combine / finalize / finalize_batch / prefix_combine / elements / txs get edge values and
sizes on both sides of every chunk, block and kernel switch.  Inverses are pow(d, -1, p) (0 for d = 0 mod p)."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

import u3072_model as um

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
P, ONES, PD = um.P, um.ONES, um.PRIME_DIFF
KGV_ERR_ARG = -1
SCAN_SIZES = (1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1025)  # KGV_SCAN_CHUNK = 32, 8 groups per block


def le(x):
    return x.to_bytes(384, "little")


def val(b):
    return int.from_bytes(bytes(b), "little")


def inv(d):
    return pow(d, -1, P) if d % P else 0


def fin_hash(x):
    return hashlib.blake2b(le(x), digest_size=32, key=b"MuHashFinalize").digest()


def vals_of(buf, n, pitch=384, off=0):
    b = np.asarray(buf).reshape(-1).tobytes()
    return [val(b[off + i * pitch: off + i * pitch + 384]) for i in range(n)]


@pytest.fixture(scope="module")
def ctx():
    import rusty_kaspa_b200 as rk
    c = rk.GpuContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    return json.load(open(os.path.join(HERE, "golden", "muhash.json")))["u3072_edges"]


def _to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sync(ctx):
    import torch
    torch.cuda.synchronize()
    assert ctx._lib.kgv_synchronize(ctx._h) == 0


# ---------------------------------------------------------------------------------------------- the two multipliers
def level(ctx, coop, vals):
    inp = np.frombuffer(b"".join(le(v) for v in vals), dtype=np.uint8).copy()
    h = (len(vals) + 1) // 2
    out = np.zeros(h * 384, dtype=np.uint8)
    ctx._check(ctx._lib.kgv_debug_u3072_level(ctx._h, coop, inp.ctypes.data, len(vals), out.ctypes.data))
    return vals_of(out, h)


def test_level_kernels_return_the_exact_fold(ctx):
    """out[t] = fold(in[2t] * in[2t+1]) bit for bit (not just mod p), the odd last value copied, for the per-thread and the
    cooperative level kernel; n_in puts 1, 2, 7 and 8 groups in the last coop block (a warp with one multiplying group and one
    idle or copying group) and a partial last 128-thread block in the per-thread kernel."""
    cases = um.edge_cases()
    counts = um.flag_counts(cases)
    assert all(c >= 4 for c in counts.values()), counts
    rnd = random.Random(21)
    vals = [x for a, b, _, _ in cases for x in (a, b)]
    vals += [rnd.getrandbits(3072) for _ in range(524 - len(vals))]
    assert len(vals) == 524
    # coop: groups in the last block of 8 = 2, 2, 7, 8, 1, 1, 6, 6 for n = 499 .. 524; odd n: the last group copies (499: next to a
    # multiplying group in its warp, 513: next to an idle one; 514: one multiplying group next to an idle one)
    # per-thread: n = 257 / 258 leave one thread in the last block, 523 / 524 six
    sizes = {1: (1, 2, 3, 4, 499, 500, 510, 512, 513, 514, 523, 524), 0: (1, 2, 3, 257, 258, 523, 524)}
    for coop, ns in sizes.items():
        for n in ns:
            got = level(ctx, coop, vals[:n])
            assert len(got) == (n + 1) // 2
            for t, g in enumerate(got):
                if 2 * t + 1 < n:
                    assert g == um.fold(vals[2 * t] * vals[2 * t + 1]), (coop, n, t, hex(vals[2 * t]), hex(vals[2 * t + 1]))
                else:
                    assert g == vals[2 * t], (coop, n, t)


# ---------------------------------------------------------------------------------------------- combine / finalize
def combine(ctx, na, da, nb, db):
    bufs = [np.frombuffer(le(x), dtype=np.uint8).copy() for x in (na, da, nb, db)]
    ctx._check(ctx._lib.kgv_muhash_combine(ctx._h, *[b.ctypes.data for b in bufs]))
    return val(bufs[0]), val(bufs[1])


def finalize(ctx, num, den):
    n, d = np.frombuffer(le(num), dtype=np.uint8).copy(), np.frombuffer(le(den), dtype=np.uint8).copy()
    ser, h = np.zeros(384, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    ctx._check(ctx._lib.kgv_muhash_finalize(ctx._h, n.ctypes.data, d.ctypes.data, ser.ctypes.data, h.ctypes.data))
    return val(ser), h.tobytes()


def test_combine_edge_pairs_is_canonical_product(ctx, golden):
    cases = um.edge_cases()
    for (a, b, _, _), (c, d, _, _) in zip(cases, cases[1:] + cases[:1]):
        assert combine(ctx, a, c, b, d) == (a * b % P, c * d % P), (hex(a), hex(b), hex(c), hex(d))
    m = val(bytes.fromhex(golden["mul_max"]["a"]))  # u3072.rs test_mul_max: (p - 1)^2 = 1
    assert m == P - 1
    assert combine(ctx, m, m, m, m) == (1, 1) == (val(bytes.fromhex(golden["mul_max"]["a_times_a"])),) * 2


def test_finalize_edge_numerators_and_denominators(ctx, golden):
    rnd = random.Random(31)
    r = rnd.getrandbits(3072) % P
    nums = [0, 1, P - 1, P, P + 1, ONES, ONES - 1, 2**3071, r, P + rnd.randrange(PD), 0, 5, r]
    dens = [1, P - 1, P + 1, ONES, 2**3071, r, P + 7, ONES - 5, 1, 1, 0, P, r]  # 0 and p: 0 has inverse 0 (u3072.rs:163-165)
    for n, d in zip(nums, dens):
        want = n * inv(d) % P
        assert finalize(ctx, n, d) == (want, fin_hash(want)), (hex(n), hex(d))
    e = val(bytes.fromhex(golden["inverse_edge_case"]))  # u3072.rs test_inverse_edge_case: inverse(inverse(x)) == x
    ie, _ = finalize(ctx, 1, e)
    assert ie == inv(e) and finalize(ctx, 1, ie)[0] == e
    # u3072.rs exhuastive_test_div_overflow, at its ends: x = 2^3072 - 1 - i; x / 1 = x - p, x / x = 1 except for x = p
    for i in (0, 1, PD - 2, PD - 1):
        x = ONES - i
        assert finalize(ctx, x, 1)[0] == PD - 1 - i
        assert finalize(ctx, x, x)[0] == (0 if i == PD - 1 else 1)


def test_finalize_batch_over_overflowing_values(ctx):
    """a sample of the 1 103 717 values in [p, 2^3072): x / 1 = x - p and x / x = 1 (x = p, whose inverse is 0, excluded:
    the batch requires nonzero denominators)"""
    rnd = random.Random(41)
    idx = [0, 1, PD - 2] + rnd.sample(range(2, PD - 2), 997)
    xs = [ONES - i for i in idx]
    assert vals_of(finalize_batch(ctx, xs, [1] * len(xs), 384, False, True)[1], len(xs)) == [PD - 1 - i for i in idx]
    assert vals_of(finalize_batch(ctx, xs, xs, 768, False, True)[1], len(xs)) == [1] * len(xs)


# ---------------------------------------------------------------------------------------------- finalize_batch
def _place(nums, dens, pitch):
    """(num buffer, num offset, den buffer, den offset): pitch 768 / 1024 are (numerator || denominator) records (the denominator
    at pitch / 2), other pitches two separate arrays"""
    n = len(nums)
    if pitch in (768, 1024):
        buf = np.zeros(n * pitch, dtype=np.uint8)
        for i, (a, b) in enumerate(zip(nums, dens)):
            buf[i * pitch: i * pitch + 384] = np.frombuffer(le(a), dtype=np.uint8)
            buf[i * pitch + pitch // 2: i * pitch + pitch // 2 + 384] = np.frombuffer(le(b), dtype=np.uint8)
        return buf, 0, buf, pitch // 2
    nb, db = np.zeros(n * pitch, dtype=np.uint8), np.zeros(n * pitch, dtype=np.uint8)
    for i, (a, b) in enumerate(zip(nums, dens)):
        nb[i * pitch: i * pitch + 384] = np.frombuffer(le(a), dtype=np.uint8)
        db[i * pitch: i * pitch + 384] = np.frombuffer(le(b), dtype=np.uint8)
    return nb, 0, db, 0


def finalize_batch(ctx, nums, dens, pitch, device, want_ser):
    n = len(nums)
    nb, no, db, do = _place(nums, dens, pitch)
    lib = ctx._lib
    if device:
        import torch
        dn = _to_dev(nb)
        dd = dn if db is nb else _to_dev(db)
        h = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
        ser = torch.zeros(n * 384, dtype=torch.uint8, device="cuda") if want_ser else None
        _sync(ctx)
        rc = lib.kgv_muhash_finalize_batch(ctx._h, dn.data_ptr() + no, dd.data_ptr() + do, n, pitch, ser.data_ptr() if want_ser else None, h.data_ptr())
        assert rc == 0, lib.kgv_last_error(ctx._h)
        _sync(ctx)
        return h.cpu().numpy().reshape(n, 32), ser.cpu().numpy() if want_ser else None
    h = np.zeros((n, 32), dtype=np.uint8)
    ser = np.zeros(n * 384, dtype=np.uint8) if want_ser else None
    rc = lib.kgv_muhash_finalize_batch(ctx._h, nb.ctypes.data + no, db.ctypes.data + do, n, pitch, ser.ctypes.data if want_ser else None, h.ctypes.data)
    assert rc == 0, lib.kgv_last_error(ctx._h)
    return h, ser


def _batch_values(n_max, seed):
    """random residues, non-canonical values and edge values; numerators may be 0, denominators are never 0 mod p"""
    rnd = random.Random(seed)
    edge_n = [0, 1, P - 1, P, P + 1, ONES, ONES - 1, 2**3071, PD - 1, PD + 1]
    edge_d = [1, P - 1, P + 1, ONES, ONES - 1, 2**3071, PD - 1, PD + 1, ONES - PD + 2]
    nums = [rnd.choice(edge_n) if rnd.random() < 0.2 else rnd.getrandbits(3072) for _ in range(n_max)]
    dens = [rnd.choice(edge_d) if rnd.random() < 0.2 else rnd.getrandbits(3072) for _ in range(n_max)]
    dens = [d if d % P else d + 1 for d in dens]
    return nums, dens


def test_finalize_batch_sizes_pitches_and_pointer_kinds(ctx):
    nums, dens = _batch_values(max(SCAN_SIZES), 51)
    want = [a * inv(b) % P for a, b in zip(nums, dens)]
    want_h = [fin_hash(x) for x in want]
    for n in SCAN_SIZES:
        for pitch in (384, 768, 400, 1024):
            for device in (False, True):
                for want_ser in (False, True):
                    h, ser = finalize_batch(ctx, nums[:n], dens[:n], pitch, device, want_ser)
                    assert [bytes(r) for r in h] == want_h[:n], (n, pitch, device, want_ser)
                    if want_ser:
                        assert vals_of(ser, n) == want[:n], (n, pitch, device)
    for i in (0, 32, 33, 1024):  # the batch agrees with one kgv_muhash_finalize per value
        assert finalize(ctx, nums[i], dens[i]) == (want[i], want_h[i])


def test_finalize_batch_and_prefix_combine_reject_unaligned_buffers(ctx):
    """pitches that are not a multiple of 16 and misaligned device buffers give KGV_ERR_ARG before any kernel runs;
    host buffers are staged into device memory, so their alignment does not matter"""
    import torch
    lib, n = ctx._lib, 4
    one = np.zeros(n * 768 + 64, dtype=np.uint8)
    one[0: n * 768: 384] = 1  # every numerator and denominator is 1
    h = np.zeros(n * 32, dtype=np.uint8)
    for pitch in (388, 392, 776, 100, 0):
        assert lib.kgv_muhash_finalize_batch(ctx._h, one.ctypes.data, one.ctypes.data + 384, n, pitch, None, h.ctypes.data) == KGV_ERR_ARG, pitch
    d = _to_dev(one)
    dh = torch.zeros(n * 32 + 16, dtype=torch.uint8, device="cuda")
    ds = torch.zeros(n * 384 + 16, dtype=torch.uint8, device="cuda")
    _sync(ctx)
    base, hp, sp = d.data_ptr(), dh.data_ptr(), ds.data_ptr()
    for num, hh, ss in ((base + 4, hp, sp), (base + 8, hp, sp), (base, hp + 2, sp), (base, hp, sp + 2), (base, hp + 1, None)):
        assert lib.kgv_muhash_finalize_batch(ctx._h, num, num + 384, n, 768, ss, hh) == KGV_ERR_ARG, (num - base, hh - hp, ss and ss - sp)
        assert b"aligned" in lib.kgv_last_error(ctx._h)
    assert lib.kgv_muhash_prefix_combine(ctx._h, None, base + 4, n) == KGV_ERR_ARG
    assert lib.kgv_muhash_prefix_combine(ctx._h, None, base + 8, n) == KGV_ERR_ARG
    # the same buffers, aligned: accepted and right (1 / 1 = 1); 4-byte aligned hash and serialized pointers are enough
    assert lib.kgv_muhash_finalize_batch(ctx._h, base, base + 384, n, 768, sp + 4, hp + 4) == 0
    _sync(ctx)
    assert bytes(dh.cpu().numpy()[4: 4 + 32 * n]) == fin_hash(1) * n
    assert vals_of(ds.cpu().numpy()[4: 4 + 384 * n], n) == [1] * n
    hh = np.zeros(n * 32 + 4, dtype=np.uint8)  # unaligned host pointers (numerator = denominator = 2^3040)
    assert lib.kgv_muhash_finalize_batch(ctx._h, one.ctypes.data + 4, one.ctypes.data + 4, n, 768, None, hh.ctypes.data + 1) == 0
    assert bytes(hh[1: 1 + 32 * n]) == fin_hash(1) * n


# ---------------------------------------------------------------------------------------------- prefix_combine
def test_prefix_combine_sizes_inits_and_pointer_kinds(ctx):
    nums, dens = _batch_values(max(SCAN_SIZES), 61)
    inits = {None: (1, 1), "edge": (ONES, P + 1)}
    for name, (i_num, i_den) in inits.items():
        want, a, b = [], i_num, i_den
        for x, y in zip(nums, dens):
            a, b = a * x % P, b * y % P
            want.append((a, b))
        for n in SCAN_SIZES:
            recs = np.frombuffer(b"".join(le(x) + le(y) for x, y in zip(nums[:n], dens[:n])), dtype=np.uint8).copy()
            ib = None if name is None else np.frombuffer(le(i_num) + le(i_den), dtype=np.uint8).copy()
            for device in (False, True):
                if device:
                    v = _to_dev(recs)
                    di = None if ib is None else _to_dev(ib)
                    _sync(ctx)
                    rc = ctx._lib.kgv_muhash_prefix_combine(ctx._h, None if di is None else di.data_ptr(), v.data_ptr(), n)
                    assert rc == 0, ctx._lib.kgv_last_error(ctx._h)
                    _sync(ctx)
                    out = v.cpu().numpy()
                else:
                    out = recs.copy()
                    ctx._check(ctx._lib.kgv_muhash_prefix_combine(ctx._h, None if ib is None else ib.ctypes.data, out.ctypes.data, n))
                got = list(zip(vals_of(out, n, 768, 0), vals_of(out, n, 768, 384)))
                assert got == want[:n], (name, n, device)


# ---------------------------------------------------------------------------------------------- element trees
@pytest.fixture(scope="module")
def elements(oracle):
    """the MuHash elements of 32 769 byte strings: keyed BLAKE2b, then the oracle's ChaCha20 expansion"""
    import pyref
    items = [b"u3072 tree item %d" % i + bytes(i % 7) for i in range(32769)]
    out = ctypes.create_string_buffer(384)
    es = []
    for d in items:
        oracle.ok_muhash_expand(pyref.blake2b_keyed(b"MuHashElement", d), out)
        es.append(val(out.raw))
    assert [pyref.muhash_element(items[i]) for i in (0, 1, 32768)] == [es[0], es[1], es[32768]]
    return items, es


def test_elements_trees_around_the_kernel_switch(ctx, elements):
    """numerator and denominator trees of n elements, n on both sides of the level-size switch (a first level of more than
    8192 products runs the per-thread multiplier) and of the powers of two, all-add, all-remove and alternating"""
    items, es = elements
    sizes = (1, 2, 3, 16383, 16384, 16385, 16386, 32769)
    prod_all, prod_even, prod_odd, at = 1, 1, 1, {}
    for i, e in enumerate(es):
        prod_all = prod_all * e % P
        if i % 2:
            prod_odd = prod_odd * e % P
        else:
            prod_even = prod_even * e % P
        if i + 1 in sizes:
            at[i + 1] = (prod_all, prod_even, prod_odd)
    for n in sizes:
        data = np.frombuffer(b"".join(items[:n]) + bytes(8), dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(x) for x in items[:n]])
        pa, pe, po = at[n]
        for name, rem, want in (("add", np.zeros(n, np.uint8), (pa, 1)), ("remove", np.ones(n, np.uint8), (1, pa)),
                                ("alternating", (np.arange(n) % 2).astype(np.uint8), (pe, po))):
            num, den = np.zeros(384, np.uint8), np.zeros(384, np.uint8)
            ctx._check(ctx._lib.kgv_muhash_elements(ctx._h, data.ctypes.data, offs.ctypes.data, rem.ctypes.data, n, num.ctypes.data, den.ctypes.data))
            assert (val(num), val(den)) == want, (n, name)


# ---------------------------------------------------------------------------------------------- kgv_muhash_txs
class OkMuHash(ctypes.Structure):
    _fields_ = [("num", ctypes.c_uint64 * 48), ("den", ctypes.c_uint64 * 48)]


def test_txs_with_inputs_and_outputs_on_opposite_sides_of_the_switch(ctx, oracle):
    """16 385 inputs (a first denominator level of 8 193 products: per-thread multiplier) and 300 outputs (cooperative) in one
    batch, against the oracle's ok_muhash_accepted"""
    from rusty_kaspa_b200 import MuHash
    from rusty_kaspa_b200.simgen import SUBNET_NATIVE
    from rusty_kaspa_b200.txbatch import build_batch
    import oracle_tx
    n_tx, n_in = 150, 16385
    counts = [n_in // n_tx] * n_tx
    counts[-1] += n_in - sum(counts)
    spk = bytes([0x20]) + bytes(range(32)) + bytes([0xAC])
    txs, ents, k = [], [], 0
    for t, c in enumerate(counts):
        ins = [{"txid": hashlib.blake2b(b"%d" % (k + j), digest_size=32).digest(), "index": (k + j) % 3, "sigscript": b"", "sequence": 0,
                "sig_op_count": 1} for j in range(c)]
        ents.append([{"amount": 1000 + k + j, "spk_version": 0, "script": spk, "block_daa_score": 7, "is_coinbase": (k + j) % 50 == 0} for j in range(c)])
        k += c
        outs = [{"value": 500 + t, "spk_version": 0, "script": bytes([0x51])}, {"value": 1 + t, "spk_version": 0, "script": spk}]
        txs.append({"version": 0, "inputs": ins, "outputs": outs, "lock_time": 0, "subnetwork_id": SUBNET_NATIVE, "gas": 0, "payload": b"", "mass": 0})
    b = build_batch(txs, ents)
    assert len(b.inputs) == 16385 and len(b.outputs) == 300
    ob = oracle_tx.ok_batch(b)
    rng = np.random.default_rng(17)
    for accept in (np.ones(n_tx, dtype=np.uint8), (rng.random(n_tx) < 0.8).astype(np.uint8)):
        m = OkMuHash()
        oracle.ok_muhash_accepted(ctypes.byref(m), ctypes.byref(ob), b.entries.ctypes.data_as(ctypes.c_void_p), accept.ctypes.data_as(ctypes.c_void_p),
                                  ctypes.c_uint64(99))
        num, den = ctypes.create_string_buffer(384), ctypes.create_string_buffer(384)
        oracle.ok_muhash_raw(ctypes.byref(m), num, den)
        g = MuHash.from_transactions(ctx, b, accept, 99)
        assert (g.numerator, g.denominator) == (num.raw, den.raw)
