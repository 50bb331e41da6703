"""Where each caller array of a C entry point may live (include/kgv.h, Conventions; the table above class kgv_io in kgv_internal.h).

SPEC restates that table call by call.  For the calls with a builder below, every side assignment the table allows must give the
return code, the output bytes and the launch count of the all-host call, and the all-host call must equal a plain reference (the C
oracle, oracle/pyref.py or Python integers).  Every assignment the table forbids (one member of a shared group flipped, a device
pointer for a host-only argument, a host pointer for a device-only one, a misaligned device array where an alignment is documented)
must give KGV_ERR_ARG naming the call, with the outputs untouched and no launch.  Host outputs are read as soon as the call returns;
device outputs only after kgv_synchronize."""
import ctypes
import itertools
import random

import numpy as np
import pytest

KGV_ERR_ARG = -1
SENTINEL = 0xA5

# call -> the arrays that share one side ("together", one list per group), the arrays each on its own side ("own"), the arguments that
# must be host memory ("host") or device memory ("device"), and documented device alignments in bytes ("align").  "batch" stands for
# the arrays of a kgv_tx_batch, which always share one side.
SPEC = {
    "kgv_schnorr_verify": dict(together=[["pk32", "msg32", "sig64", "status"]]),
    "kgv_ecdsa_verify": dict(together=[["pk33", "msg32", "sig64", "status"]]),
    "kgv_status_to_bitmap": dict(together=[["status", "bitmap"]]),
    "kgv_tx_ids": dict(together=[["batch"]], own=["out32"]),
    "kgv_tx_hashes": dict(together=[["batch"]], own=["out32"]),
    "kgv_sighash": dict(together=[["batch"], ["items", "out32"]]),
    "kgv_merkle_roots": dict(together=[["hashes32", "roots32"]], host=["first"]),
    "kgv_block_hash_merkle_roots": dict(together=[["batch"]], own=["roots32"], host=["block_first_tx"]),
    "kgv_block_set_checks": dict(together=[["batch"]], own=["out"], host=["block_first_tx"]),
    # with device offsets, data and remove must be device memory too (see _elements_allowed)
    "kgv_muhash_elements": dict(together=[["numerator384", "denominator384"]], own=["data", "offsets", "remove"]),
    "kgv_muhash_combine": dict(own=["numerator_a", "denominator_a", "numerator_b", "denominator_b"]),
    "kgv_muhash_finalize": dict(own=["numerator384", "denominator384", "serialized384", "hash32"]),
    "kgv_muhash_finalize_batch": dict(together=[["numerators384", "denominators384", "hashes32"]], own=["serialized384"],
                                      align={"numerators384": 16, "hashes32": 4, "serialized384": 4}),
    "kgv_muhash_prefix_combine": dict(own=["values768", "init768"], align={"values768": 16}),
    "kgv_muhash_txs": dict(together=[["batch"], ["numerator384", "denominator384"]], own=["accept"]),
    "kgv_utxo_muhash": dict(own=["numerator384"]),
    "kgv_utxo_lookup": dict(own=["keys36", "entries", "scripts_out", "found"]),
    "kgv_utxo_apply_diff": dict(own=["rem_keys36", "rem_status", "add_keys36", "add_entries", "add_bytes", "add_status"]),
    "kgv_utxo_export": dict(own=["keys36", "entries", "bytes"], host=["n_out", "bytes_out"]),
    "kgv_utxo_count": dict(host=["count"]),
    "kgv_utxo_digest": dict(host=["out32"]),
    "kgv_utxo_stats": dict(host=["out"]),
    "kgv_sigcache_counters": dict(host=["hits", "inserts", "lookups", "evictions"]),
    "kgv_utxo_import_chunk": dict(own=["keys36", "entries", "bytes"], host=["numerator384"]),
    "kgv_utxo_apply_accepted": dict(together=[["batch"]], own=["accept"]),
    "kgv_validate_txs": dict(together=[["batch"]], own=["results"], host=["params"]),
    "kgv_validate_populated": dict(together=[["batch"]], own=["results"], host=["params"]),
    "kgv_validate_mempool_txs": dict(together=[["results", "batch", "args", "storage_mass", "entries_out", "scripts_out"]],
                                     host=["params", "scripts_used"]),
    "kgv_validate_mempool_txs_in_parallel": dict(together=[["results", "batch", "args", "storage_mass", "masses", "entries_out", "scripts_out"]],
                                                 host=["params", "rules", "scripts_used"]),
    "kgv_validate_mempool_txs_with_policy": dict(together=[["results", "batch", "args", "storage_mass", "masses", "entries_out", "scripts_out",
                                                            "detail"]], host=["params", "rules", "policy", "scripts_used"]),
    "kgv_validate_txs_in_isolation": dict(together=[["results", "batch", "masses"]], host=["rules"]),
    "kgv_check_txs_standard_in_isolation": dict(together=[["results", "batch", "masses", "detail"]], host=["policy"]),
    "kgv_check_txs_standard_in_context": dict(together=[["results", "batch", "masses", "storage_mass", "fee", "detail"]], host=["policy"]),
    "kgv_outputs_dust": dict(together=[["is_dust", "batch"]]),
    "kgv_validate_block_bodies": dict(together=[["results", "batch", "headers", "masses", "roots32"]],
                                      host=["block_first_tx", "rules", "body_rules"]),
    "kgv_hash_headers": dict(together=[["headers", "parents32", "level_len", "hash32", "pre_pow32"]],
                             align={"headers": 8, "parents32": 8, "level_len": 4, "hash32": 8, "pre_pow32": 8}),
    "kgv_validate_headers_in_isolation": dict(together=[["headers", "parents32", "level_len", "results", "hash32", "pow32"]], host=["rules"],
                                              align={"headers": 8, "parents32": 8, "level_len": 4, "results": 8, "hash32": 8, "pow32": 8}),
    "kgv_replay_window": dict(together=[["batch"]], own=["results", "accept"], host=["blocks", "params", "stats"]),
    "kgv_replay_muhash": dict(own=["values768"], host=["group_first_block"]),
    "kgv_replay_diffs": dict(together=[["ranges", "rem_keys36", "rem_entries", "add_keys36", "add_entries", "bytes"]],
                             host=["group_first_block", "n_rem_out", "n_add_out", "bytes_out"], align={"rem_entries": 8, "add_entries": 8}),
    "kgv_replay_verify_chain": dict(together=[["results", "headers", "merged_flags", "init768", "block_fees", "multisets768"]],
                                    host=["group_first_block", "rules", "body_rules"]),
    "kgv_check_scripts": dict(together=[["batch"]], own=["tx_indices", "results"]),
    "kgv_shard_allgather": dict(device=["local_shard", "all_shards"]),
    "kgv_shard_publish_bitmap": dict(device=["status"], host=["epoch_out"]),
    "kgv_shard_publish_bytes": dict(device=["src"], host=["epoch_out"]),
    "kgv_shard_wait": dict(device=["all_shards"]),
}


def _elements_allowed(sides):
    return sides["offsets"] == "h" or (sides["data"] == "d" and sides["remove"] == "d")


ALLOWED_EXTRA = {"kgv_muhash_elements": _elements_allowed}


def allowed_assignments(call, names):
    """every side assignment SPEC allows for the arrays `names` of `call`: one side per shared group, one per own array"""
    s = SPEC[call]
    units = [[n for n in g if n in names] for g in s.get("together", [])] + [[n] for n in s.get("own", []) if n in names]
    units = [u for u in units if u]
    fixed = {n: "h" for n in s.get("host", []) if n in names}
    fixed.update({n: "d" for n in s.get("device", []) if n in names})
    out = []
    for combo in itertools.product("hd", repeat=len(units)):
        sides = dict(fixed)
        for u, side in zip(units, combo):
            sides.update({n: side for n in u})
        if ALLOWED_EXTRA.get(call, lambda _: True)(sides):
            out.append(sides)
    return out


def forbidden_assignments(call, names):
    """one member of each shared group flipped (from all-host and from all-device), each host-only argument on the device, each
    device-only argument on the host, and the conditional rules of ALLOWED_EXTRA"""
    s = SPEC[call]
    host_fixed = {n: "h" for n in s.get("host", []) if n in names}
    dev_fixed = {n: "d" for n in s.get("device", []) if n in names}
    free = [n for n in names if n not in host_fixed and n not in dev_fixed]
    out = []
    for g in s.get("together", []):
        g = [n for n in g if n in names]
        if len(g) < 2:
            continue
        for base in "hd":
            sides = {n: base for n in free}
            sides.update(host_fixed)
            sides.update(dev_fixed)
            sides[g[0]] = "d" if base == "h" else "h"
            out.append(sides)
    for n in host_fixed:
        sides = {m: "h" for m in free}
        sides.update(host_fixed)
        sides.update(dev_fixed)
        sides[n] = "d"
        out.append(sides)
    for n in dev_fixed:
        sides = {m: "h" for m in free}
        sides.update(host_fixed)
        sides.update(dev_fixed)
        sides[n] = "h"
        out.append(sides)
    if call in ALLOWED_EXTRA:
        for combo in itertools.product("hd", repeat=len(free)):
            sides = dict(zip(free, combo))
            sides.update(host_fixed)
            if not ALLOWED_EXTRA[call](sides):
                out.append(sides)
    return out


# ---------------------------------------------------------------------------------------------
# running one call with its arrays on given sides
# ---------------------------------------------------------------------------------------------
class Case:
    """arrays: name -> (uint8 numpy array, kind) with kind "in", "out" or "inout" ("batch.txs" and the like are the arrays of the
    transaction batch, which take the side of "batch"); invoke(ptrs) -> rc; extra() -> bytes of state the call
    changes outside its arrays (a table digest), read after the call; close() frees what the case created"""

    def __init__(self, arrays, invoke, extra=None, close=None):
        self.arrays, self.invoke, self.extra, self.close = arrays, invoke, extra, close


def _place(data, side, misalign, keep):
    """a copy of data on the host or the device, starting `misalign` bytes past a 256-byte boundary; returns (ptr, reader)"""
    import torch
    n = len(data)
    if side == "h":
        raw = np.empty(n + 512, dtype=np.uint8)
        off = (-raw.ctypes.data) % 256 + misalign
        view = raw[off:off + n]
        view[:] = data
        keep.append(raw)
        return view.ctypes.data, lambda: view.tobytes()
    t = torch.empty(n + 512, dtype=torch.uint8, device="cuda")
    keep.append(t)
    if n:
        t[misalign:misalign + n].copy_(torch.from_numpy(np.ascontiguousarray(data)))
    return t.data_ptr() + misalign, lambda: t[misalign:misalign + n].cpu().numpy().tobytes()


def run(ctx, case, sides, misalign=None):
    """-> (rc, launches, {output name: bytes}, extra, last error).  Host outputs are read straight after the call, device outputs after
    kgv_synchronize."""
    lib, h = ctx._lib, ctx._h
    keep, ptrs, readers = [], {}, {}
    side = lambda name: sides.get(name.split(".")[0], "h")
    for name, (data, kind) in case.arrays.items():
        init = np.full(len(data), SENTINEL, dtype=np.uint8) if kind == "out" else data
        ptrs[name], rd = _place(init, side(name), (misalign or {}).get(name, 0), keep)
        if kind != "in":
            readers[name] = rd
    before = lib.kgv_launch_count(h)
    rc = case.invoke(ptrs)
    err = lib.kgv_last_error(h).decode() if rc else ""
    outs = {n: rd() for n, rd in readers.items() if side(n) == "h"}  # no synchronisation before these
    assert lib.kgv_synchronize(h) == 0
    outs.update({n: rd() for n, rd in readers.items() if side(n) == "d"})
    launches = lib.kgv_launch_count(h) - before
    extra = case.extra() if case.extra else b""
    return rc, launches, outs, extra, err


def initial_outputs(case):
    return {n: (bytes([SENTINEL]) * len(d) if k == "out" else d.tobytes()) for n, (d, k) in case.arrays.items() if k != "in"}


def check_matrix(ctx, call, make, anchor):
    """make() -> Case (fresh state per run); anchor(outs, extra) asserts the all-host result against the plain reference.
    Returns the number of (call, assignment) cases run."""
    names = list(make_names(make))
    base_case = make()
    rc0, n0, out0, ex0, err0 = run(ctx, base_case, {n: "h" for n in names})
    if base_case.close:
        base_case.close()
    assert rc0 == 0, (call, err0)
    anchor(out0, ex0)
    count = 1
    for sides in allowed_assignments(call, names):
        c = make()
        rc, n, out, ex, err = run(ctx, c, sides)
        if c.close:
            c.close()
        assert (rc, n) == (rc0, n0), (call, sides, err)
        assert out == out0, (call, sides, [k for k in out if out[k] != out0[k]])
        assert ex == ex0, (call, sides)
        count += 1
    for sides in forbidden_assignments(call, names):
        c = make()
        rc, n, out, ex, err = run(ctx, c, sides)
        if c.close:
            c.close()
        assert rc == KGV_ERR_ARG, (call, sides, rc)
        assert call in err, (call, sides, err)
        assert n == 0, (call, sides)
        assert out == initial_outputs(c), (call, sides)
        count += 1
    return count


def make_names(make):
    c = make()
    names = list(dict.fromkeys(n.split(".")[0] for n in c.arrays))
    if c.close:
        c.close()
    return names


def u8(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()


# ---------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------
def _pyref():
    import pyref
    return pyref


def _rand_residue(rnd):
    return rnd.randrange(1, _pyref().MUHASH_P)


def _le(x):
    return x.to_bytes(384, "little")


def _muhash_combine(ctx):
    rnd = random.Random(11)
    P = _pyref().MUHASH_P
    # edges: a value just below p, 1, and two random residues
    na, da, nb, db = P - 1, 1, _rand_residue(rnd), _rand_residue(rnd)
    arr = lambda x: np.frombuffer(_le(x), dtype=np.uint8).copy()

    def make():
        a = {"numerator_a": (arr(na), "inout"), "denominator_a": (arr(da), "inout"), "numerator_b": (arr(nb), "in"),
             "denominator_b": (arr(db), "in")}
        return Case(a, lambda p: ctx._lib.kgv_muhash_combine(ctx._h, p["numerator_a"], p["denominator_a"], p["numerator_b"], p["denominator_b"]))

    def anchor(out, _):
        assert out["numerator_a"] == _le(na * nb % P) and out["denominator_a"] == _le(da * db % P)
    return make, anchor


def _muhash_finalize(ctx):
    rnd = random.Random(12)
    pr = _pyref()
    num, den = _rand_residue(rnd), pr.MUHASH_P - 2
    arr = lambda x: np.frombuffer(_le(x), dtype=np.uint8).copy()

    def make():
        a = {"numerator384": (arr(num), "in"), "denominator384": (arr(den), "in"), "serialized384": (np.zeros(384, np.uint8), "out"),
             "hash32": (np.zeros(32, np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_muhash_finalize(ctx._h, p["numerator384"], p["denominator384"], p["serialized384"], p["hash32"]))

    def anchor(out, _):
        m = pr.MuHash()
        m.num, m.den = num, den
        ser = _le(num * pow(den, pr.MUHASH_P - 2, pr.MUHASH_P) % pr.MUHASH_P)
        assert out["serialized384"] == ser and out["hash32"] == m.finalize()
    return make, anchor


def _elements_data(n=9, seed=13):
    rnd = random.Random(seed)
    items = [bytes(rnd.randrange(256) for _ in range(rnd.choice([0, 1, 31, 32, 33, 64, 200]))) for _ in range(n)]
    rem = np.array([rnd.random() < 0.4 for _ in range(n)], dtype=np.uint8)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(d) for d in items])
    data = np.frombuffer(b"".join(items) + b"\0", dtype=np.uint8).copy()  # one spare byte: never an empty array
    return items, rem, offs, data


def _muhash_elements(ctx, n=9, seed=13):
    pr = _pyref()
    items, rem, offs, data = _elements_data(n, seed)

    def make():
        a = {"data": (data, "in"), "offsets": (u8(offs), "in"), "remove": (rem.copy(), "in"), "numerator384": (np.zeros(384, np.uint8), "out"),
             "denominator384": (np.zeros(384, np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_muhash_elements(ctx._h, p["data"], p["offsets"], p["remove"], n, p["numerator384"], p["denominator384"]))

    def anchor(out, _):
        m = pr.MuHash()
        for d, r in zip(items, rem):
            (m.remove_element if r else m.add_element)(d)
        assert out["numerator384"] == _le(m.num) and out["denominator384"] == _le(m.den)
    return make, anchor


def _records(n, seed):
    rnd = random.Random(seed)
    return [(_rand_residue(rnd), _rand_residue(rnd)) for _ in range(n)]


def _muhash_finalize_batch(ctx, n=37):
    pr = _pyref()
    recs = _records(n, 14)
    nums = np.frombuffer(b"".join(_le(a) for a, _ in recs), dtype=np.uint8).copy()
    dens = np.frombuffer(b"".join(_le(b) for _, b in recs), dtype=np.uint8).copy()

    def make():
        a = {"numerators384": (nums, "in"), "denominators384": (dens, "in"), "serialized384": (np.zeros(n * 384, np.uint8), "out"),
             "hashes32": (np.zeros(n * 32, np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_muhash_finalize_batch(ctx._h, p["numerators384"], p["denominators384"], n, 384, p["serialized384"],
                                                                    p["hashes32"]))

    def anchor(out, _):
        ser, hs = b"", b""
        for a, b in recs:
            m = pr.MuHash()
            m.num, m.den = a, b
            hs += m.finalize()
            ser += _le(m.num)
        assert out["serialized384"] == ser and out["hashes32"] == hs
    return make, anchor


def _muhash_prefix_combine(ctx, n=40):
    P = _pyref().MUHASH_P
    recs = _records(n, 15)
    init = _records(1, 16)[0]
    vals = np.frombuffer(b"".join(_le(a) + _le(b) for a, b in recs), dtype=np.uint8).copy()
    init768 = np.frombuffer(_le(init[0]) + _le(init[1]), dtype=np.uint8).copy()

    def make():
        a = {"values768": (vals, "inout"), "init768": (init768, "in")}
        return Case(a, lambda p: ctx._lib.kgv_muhash_prefix_combine(ctx._h, p["init768"], p["values768"], n))

    def anchor(out, _):
        a, b, want = init[0], init[1], b""
        for x, y in recs:
            a, b = a * x % P, b * y % P
            want += _le(a) + _le(b)
        assert out["values768"] == want
    return make, anchor


def _status_to_bitmap(ctx, n=77):
    st = np.random.default_rng(17).integers(0, 4, n).astype(np.uint8)

    def make():
        a = {"status": (st, "in"), "bitmap": (np.zeros((n + 7) // 8, np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_status_to_bitmap(ctx._h, p["status"], n, p["bitmap"]))

    def anchor(out, _):
        assert out["bitmap"] == np.packbits((st == 1).astype(np.uint8), bitorder="little").tobytes()
    return make, anchor


def _verify(ctx, oracle, ecdsa, n=96):
    from rusty_kaspa_b200 import workload as W
    import conftest
    gen = W.ecdsa_triples if ecdsa else W.schnorr_triples
    pk, msg, sig, _ = gen(n, seed=21, n_keys=16, n_nonces=32, frac_bitflip=0.1, frac_adversarial=0.1)
    pkn = "pk33" if ecdsa else "pk32"
    fn = ctx._lib.kgv_ecdsa_verify if ecdsa else ctx._lib.kgv_schnorr_verify

    def make():
        a = {pkn: (u8(pk), "in"), "msg32": (u8(msg), "in"), "sig64": (u8(sig), "in"), "status": (np.zeros(n, np.uint8), "out")}
        return Case(a, lambda p: fn(ctx._h, p[pkn], p["msg32"], p["sig64"], n, p["status"]))

    def anchor(out, _):
        want = (conftest.oracle_ecdsa_batch if ecdsa else conftest.oracle_schnorr_batch)(oracle, pk, msg, sig)
        assert out["status"] == want.tobytes()
    return make, anchor


def _merkle_roots(ctx):
    pr = _pyref()
    rnd = random.Random(18)
    sizes = [0, 1, 2, 3, 5, 8, 9]
    first = np.zeros(len(sizes) + 1, dtype=np.uint32)
    first[1:] = np.cumsum(sizes)
    hashes = [bytes(rnd.randrange(256) for _ in range(32)) for _ in range(int(first[-1]))]
    hb = np.frombuffer(b"".join(hashes), dtype=np.uint8).copy()

    def make():
        a = {"hashes32": (hb, "in"), "first": (u8(first), "in"), "roots32": (np.zeros(32 * len(sizes), np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_merkle_roots(ctx._h, p["hashes32"], p["first"], len(sizes), p["roots32"]))

    def anchor(out, _):
        assert out["roots32"] == b"".join(pr.merkle_root(hashes[first[g]:first[g + 1]]) for g in range(len(sizes)))
    return make, anchor


def _utxo_chunk(n=24, seed=19, bad_script=False):
    """n (key, entry) pairs over one script arena; bad_script: the last entry's script runs one byte past the arena"""
    from rusty_kaspa_b200.txbatch import ENTRY_DTYPE
    rnd = random.Random(seed)
    keys = np.zeros((n, 36), dtype=np.uint8)
    ent = np.zeros(n, dtype=ENTRY_DTYPE)
    arena, scripts = b"", []
    for i in range(n):
        keys[i, :32] = np.frombuffer(bytes(rnd.randrange(256) for _ in range(32)), dtype=np.uint8)
        keys[i, 32:] = np.frombuffer(rnd.choice([0, 1, 255, 0xFFFFFFFF]).to_bytes(4, "little"), dtype=np.uint8)
        s = bytes(rnd.randrange(256) for _ in range(rnd.choice([0, 1, 34, 35, 70])))
        ent[i]["amount"], ent[i]["block_daa_score"] = rnd.randrange(1 << 50), rnd.randrange(1 << 40)
        ent[i]["script_off"], ent[i]["script_len"] = len(arena), len(s)
        ent[i]["spk_version"], ent[i]["is_coinbase"] = rnd.choice([0, 1]), rnd.choice([0, 1])
        arena += s
        scripts.append(s)
    arena_arr = np.frombuffer(arena + b"\0", dtype=np.uint8).copy()
    n_bytes = len(arena)
    if bad_script:
        ent[n - 1]["script_len"] = n_bytes - int(ent[n - 1]["script_off"]) + 1
    return keys, ent, arena_arr, n_bytes, scripts


def _utxo_import_chunk(ctx, n=24, seed=19):
    import rusty_kaspa_b200 as rk
    pr = _pyref()
    keys, ent, arena, n_bytes, scripts = _utxo_chunk(n, seed)
    start = _records(1, 20)[0][0]

    def make():
        us = rk.GpuUtxoSet(ctx, 1 << 10)
        a = {"keys36": (u8(keys), "in"), "entries": (u8(ent), "in"), "bytes": (arena, "in"),
             "numerator384": (np.frombuffer(_le(start), dtype=np.uint8).copy(), "inout")}
        return Case(a, lambda p: ctx._lib.kgv_utxo_import_chunk(ctx._h, us._h, p["keys36"], p["entries"], p["bytes"], n_bytes, n, p["numerator384"]),
                    extra=lambda: us.digest(), close=us.close)

    def anchor(out, _):
        num = start
        for i in range(n):
            e = ent[i]
            num = num * pr.muhash_element(pr.utxo_element_bytes(keys[i, :32].tobytes(), int.from_bytes(keys[i, 32:].tobytes(), "little"),
                                                                int(e["block_daa_score"]), int(e["amount"]), int(e["is_coinbase"]),
                                                                int(e["spk_version"]), scripts[i])) % pr.MUHASH_P
        assert out["numerator384"] == _le(num)
    return make, anchor


def _utxo_lookup(ctx, n=24, seed=22, stride=80):
    import rusty_kaspa_b200 as rk
    keys, ent, arena, n_bytes, scripts = _utxo_chunk(n, seed)
    us = rk.GpuUtxoSet(ctx, 1 << 10)
    one = np.frombuffer(_le(1), dtype=np.uint8).copy()
    assert ctx._lib.kgv_utxo_import_chunk(ctx._h, us._h, keys.ctypes.data, ent.ctypes.data, arena.ctypes.data, n_bytes, n - 4, one.ctypes.data) == 0
    # the last four keys are absent

    def make():
        a = {"keys36": (u8(keys), "in"), "entries": (np.zeros(n * 32, np.uint8), "out"), "scripts_out": (np.zeros(n * stride, np.uint8), "out"),
             "found": (np.zeros(n, np.uint8), "out")}
        return Case(a, lambda p: ctx._lib.kgv_utxo_lookup(ctx._h, us._h, p["keys36"], n, p["entries"], p["scripts_out"], stride, p["found"]))

    def anchor(out, _):
        from rusty_kaspa_b200.txbatch import ENTRY_DTYPE
        found = np.frombuffer(out["found"], dtype=np.uint8)
        assert found.tolist() == [1] * (n - 4) + [0] * 4
        got = np.frombuffer(out["entries"], dtype=ENTRY_DTYPE)
        sc = np.frombuffer(out["scripts_out"], dtype=np.uint8).reshape(n, stride)
        for i in range(n - 4):
            for f in ("amount", "block_daa_score", "script_len", "spk_version", "is_coinbase"):
                assert got[i][f] == ent[i][f], (i, f)
            assert sc[i, :len(scripts[i])].tobytes() == scripts[i], i
    return make, anchor, us


def _batch_arrays(b):
    """the arrays of a txbatch.TxBatch as "batch.*" case arrays"""
    a = {"batch.txs": (u8(b.txs), "in"), "batch.inputs": (u8(b.inputs), "in"), "batch.outputs": (u8(b.outputs), "in"),
         "batch.bytes": (u8(b.arena), "in")}
    if b.entries is not None:
        a["batch.entries"] = (u8(b.entries), "in")
    return a


def _c_batch(b, p):
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    return _KgvTxBatch(p["batch.txs"], len(b.txs), p["batch.inputs"], len(b.inputs), p["batch.outputs"], len(b.outputs), p.get("batch.entries"),
                       p["batch.bytes"], len(b.arena))


def _tx_digests(ctx, oracle, hashes):
    import oracle_tx
    b, _, _, _ = _window()
    fn = ctx._lib.kgv_tx_hashes if hashes else ctx._lib.kgv_tx_ids

    def make():
        a = dict(_batch_arrays(b), out32=(np.zeros(32 * len(b.txs), np.uint8), "out"))
        return Case(a, lambda p: fn(ctx._h, ctypes.byref(_c_batch(b, p)), p["out32"]))

    def anchor(out, _):
        assert out["out32"] == (oracle_tx.tx_hashes if hashes else oracle_tx.tx_ids)(oracle, b).tobytes()
    return make, anchor


def _replay_window(ctx, oracle):
    """a fresh table per run; results and accept each on their own side (a host accept beside device results included)"""
    import oracle_tx
    from rusty_kaspa_b200 import Params
    from rusty_kaspa_b200.replay import DagReplayer
    from rusty_kaspa_b200.validator import RESULT_DTYPE
    b, blocks, first, C = _window()
    nt, nb = len(b.txs), len(blocks)
    params = Params(coinbase_maturity=3, storage_mass_parameter=C)

    def make():
        rp = DagReplayer(ctx, params, 1 << 12)
        a = dict(_batch_arrays(b), blocks=(u8(blocks), "in"), params=(np.frombuffer(bytes(rp.tv.params), np.uint8).copy(), "in"),
                 stats=(np.zeros(64, np.uint8), "in"),  # written by the call, but it holds timings: not compared
                 results=(np.zeros(nt * RESULT_DTYPE.itemsize, np.uint8), "out"), accept=(np.zeros(nt, np.uint8), "out"))
        return Case(a, lambda p: ctx._lib.kgv_replay_window(ctx._h, rp.us._h, ctypes.byref(_c_batch(b, p)), p["blocks"], nb, p["params"], p["results"],
                                                            p["accept"], p["stats"]),
                    extra=lambda: rp.us.digest(), close=rp.close)

    def anchor(out, digest):
        ost = oracle_tx.State(oracle)
        exp, eacc = oracle_tx.state_replay(ost, b, first, blocks["pov_daa_score"], oracle_tx.params(coinbase_maturity=3, storage_mass_parameter=C))
        got = np.frombuffer(out["results"], dtype=RESULT_DTYPE)
        for f in ("status", "script_err"):
            assert (got[f] == exp[f]).all(), f
        ok = exp["status"] == 0
        assert (got["fee"][ok] == exp["fee"][ok]).all()
        assert out["accept"] == eacc.tobytes() and digest == ost.digest()
        ost.close()
    return make, anchor


def _headers(ctx, validate, n=40):
    import oracle_header as oh
    from rusty_kaspa_b200.headers import HeaderBatch
    params, hdrs = oh.fixture_headers(oh.FIXTURES[0])
    hb = HeaderBatch.from_dicts(hdrs[:n])
    rules = oh.fixture_rules(params, skip_pow=False)
    lib = ctx._lib
    arrays = lambda: {"headers": (u8(hb.headers), "in"), "parents32": (u8(hb.parents), "in"), "level_len": (u8(hb.level_len), "in")}
    np_, nl = len(hb.parents), len(hb.level_len)

    def make():
        a = arrays()
        a["hash32"] = (np.zeros(32 * n, np.uint8), "out")
        if validate:
            a.update(rules=(np.frombuffer(bytes(rules), np.uint8).copy(), "in"), results=(np.zeros(24 * n, np.uint8), "out"),
                     pow32=(np.zeros(32 * n, np.uint8), "out"))
            return Case(a, lambda p: lib.kgv_validate_headers_in_isolation(ctx._h, p["headers"], n, p["parents32"], np_, p["level_len"], nl, p["rules"],
                                                                           p["results"], p["hash32"], p["pow32"]))
        a["pre_pow32"] = (np.zeros(32 * n, np.uint8), "out")
        return Case(a, lambda p: lib.kgv_hash_headers(ctx._h, p["headers"], n, p["parents32"], np_, p["level_len"], nl, p["hash32"], p["pre_pow32"]))

    def anchor(out, _):
        assert out["hash32"] == b"".join(h["hash"] for h in hdrs[:n])  # the reference's own block hashes
        res, hs, pw, pre = oh.oracle_validate(oh.c_oracle(), hb, rules)
        if validate:
            assert out["results"] == res.tobytes() and out["pow32"] == pw.tobytes()
        else:
            assert out["pre_pow32"] == pre.tobytes()
    return make, anchor


def _utxo_muhash(ctx, n=24, seed=24):
    import rusty_kaspa_b200 as rk
    pr = _pyref()
    keys, ent, arena, n_bytes, scripts = _utxo_chunk(n, seed)
    us = rk.GpuUtxoSet(ctx, 1 << 10)
    one = np.frombuffer(_le(1), dtype=np.uint8).copy()
    assert ctx._lib.kgv_utxo_import_chunk(ctx._h, us._h, keys.ctypes.data, ent.ctypes.data, arena.ctypes.data, n_bytes, n, one.ctypes.data) == 0

    def make():
        return Case({"numerator384": (np.zeros(384, np.uint8), "out")}, lambda p: ctx._lib.kgv_utxo_muhash(ctx._h, us._h, p["numerator384"]))

    def anchor(out, _):
        m = pr.MuHash()
        for i in range(n):
            e = ent[i]
            m.add_element(pr.utxo_element_bytes(keys[i, :32].tobytes(), int.from_bytes(keys[i, 32:].tobytes(), "little"), int(e["block_daa_score"]),
                                                int(e["amount"]), int(e["is_coinbase"]), int(e["spk_version"]), scripts[i]))
        assert out["numerator384"] == _le(m.num)
    return make, anchor, us


BUILDERS = ["kgv_status_to_bitmap", "kgv_schnorr_verify", "kgv_ecdsa_verify", "kgv_merkle_roots", "kgv_muhash_elements", "kgv_muhash_combine",
            "kgv_muhash_finalize", "kgv_muhash_finalize_batch", "kgv_muhash_prefix_combine", "kgv_utxo_lookup", "kgv_utxo_import_chunk",
            "kgv_utxo_muhash", "kgv_tx_ids", "kgv_tx_hashes", "kgv_replay_window", "kgv_hash_headers", "kgv_validate_headers_in_isolation"]

# the calls of SPEC without a side matrix here, and what covers them instead
_REFUSALS_ONLY = "no side matrix yet: its host-only arguments are refused in test_host_only_arguments_refused"
NO_MATRIX = {
    "kgv_sighash": "no side matrix yet; its one-sided form is checked against the oracle in test_gpu_hashing",
    "kgv_block_hash_merkle_roots": _REFUSALS_ONLY,
    "kgv_block_set_checks": _REFUSALS_ONLY,
    "kgv_muhash_txs": "no side matrix yet; host and device batches are compared in test_gpu_muhash",
    "kgv_utxo_apply_diff": "no side matrix yet; it runs inside every kgv_utxo_import_chunk case of the matrix on device stand-ins",
    "kgv_utxo_export": _REFUSALS_ONLY,
    "kgv_utxo_apply_accepted": "no side matrix yet; its batch is covered by test_gpu_batch_residency",
    "kgv_validate_txs": _REFUSALS_ONLY,
    "kgv_validate_populated": _REFUSALS_ONLY,
    "kgv_validate_mempool_txs": _REFUSALS_ONLY,
    "kgv_validate_mempool_txs_in_parallel": _REFUSALS_ONLY,
    "kgv_validate_mempool_txs_with_policy": _REFUSALS_ONLY,
    "kgv_validate_txs_in_isolation": _REFUSALS_ONLY,
    "kgv_check_txs_standard_in_isolation": _REFUSALS_ONLY,
    "kgv_check_txs_standard_in_context": _REFUSALS_ONLY,
    "kgv_outputs_dust": "no side matrix yet; one shared group, whose one-sided forms are compared in test_gpu_standard",
    "kgv_validate_block_bodies": _REFUSALS_ONLY,
    "kgv_replay_muhash": "needs the state of a replay window: its host-only argument is refused in test_replay_follow_ups_refuse_device_host_arguments",
    "kgv_replay_diffs": "needs the state of a replay window: host-only arguments and entry alignment in test_replay_follow_ups_refuse_device_host_arguments",
    "kgv_replay_verify_chain": "needs the state of a replay window: host-only arguments in test_replay_follow_ups_refuse_device_host_arguments",
    "kgv_check_scripts": "no side matrix yet; its index range is refused on either side in test_check_scripts_index_range_refused_on_either_side",
    "kgv_shard_allgather": "device arrays only: refused host arrays in test_device_only_arguments_refused",
    "kgv_shard_publish_bitmap": "device arrays only: refusals in test_device_only_arguments_refused",
    "kgv_shard_publish_bytes": "device arrays only: refusals in test_device_only_arguments_refused",
    "kgv_shard_wait": "device arrays only: refusals in test_device_only_arguments_refused",
    "kgv_utxo_count": "a host result only: refused on the device in test_scalar_results_are_host_only",
    "kgv_utxo_digest": "a host result only: refused on the device in test_scalar_results_are_host_only",
    "kgv_utxo_stats": "a host result only: refused on the device in test_scalar_results_are_host_only",
    "kgv_sigcache_counters": "host results only: refused on the device in test_scalar_results_are_host_only",
}


@pytest.fixture(scope="module")
def ctx():
    import rusty_kaspa_b200 as rk
    c = rk.GpuContext(0)
    yield c
    c.close()


def _builder(ctx, oracle, call):
    """-> (make, anchor, object to close afterwards or None)"""
    if call == "kgv_utxo_lookup":
        return _utxo_lookup(ctx)
    if call == "kgv_utxo_muhash":
        return _utxo_muhash(ctx)
    if call in ("kgv_schnorr_verify", "kgv_ecdsa_verify"):
        return _verify(ctx, oracle, call == "kgv_ecdsa_verify") + (None,)
    if call in ("kgv_tx_ids", "kgv_tx_hashes"):
        return _tx_digests(ctx, oracle, call == "kgv_tx_hashes") + (None,)
    if call == "kgv_replay_window":
        return _replay_window(ctx, oracle) + (None,)
    if call in ("kgv_hash_headers", "kgv_validate_headers_in_isolation"):
        return _headers(ctx, call == "kgv_validate_headers_in_isolation") + (None,)
    return {"kgv_status_to_bitmap": _status_to_bitmap, "kgv_merkle_roots": _merkle_roots, "kgv_muhash_elements": _muhash_elements,
            "kgv_muhash_combine": _muhash_combine, "kgv_muhash_finalize": _muhash_finalize, "kgv_muhash_finalize_batch": _muhash_finalize_batch,
            "kgv_muhash_prefix_combine": _muhash_prefix_combine, "kgv_utxo_import_chunk": _utxo_import_chunk}[call](ctx) + (None,)


@pytest.mark.gpu
@pytest.mark.parametrize("call", BUILDERS)
def test_every_assignment(ctx, oracle, call):
    """the all-host call equals the plain reference; every allowed assignment gives its code, bytes and launches; every forbidden one
    is refused untouched"""
    make, anchor, extra = _builder(ctx, oracle, call)
    n = check_matrix(ctx, call, make, anchor)
    print("%s: %d (call, assignment) cases" % (call, n))
    if extra is not None:
        extra.close()


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["kgv_muhash_finalize_batch", "kgv_muhash_prefix_combine", "kgv_hash_headers", "kgv_validate_headers_in_isolation"])
def test_documented_alignment(ctx, oracle, call):
    """a device array off its documented alignment by 1, 4 or 8 bytes is refused; the same data from a host array that far off is staged
    and gives the anchor bytes"""
    make, anchor, _ = _builder(ctx, oracle, call)
    names = make_names(make)
    host = SPEC[call].get("host", [])
    for name, al in SPEC[call]["align"].items():
        for off in (1, 4, 8):
            dev = {n: ("h" if n in host else "d") for n in names}
            c = make()
            rc, n, out, _, err = run(ctx, c, dev, {name: off})
            if off % al:
                assert rc == KGV_ERR_ARG and call in err and n == 0 and out == initial_outputs(c), (name, off, rc, err)
            else:
                assert rc == 0, (name, off, err)
                anchor(out, b"")
            c = make()
            rc, n, out, _, err = run(ctx, c, {n: "h" for n in names}, {name: off})
            assert rc == 0, (name, off, err)
            anchor(out, b"")


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["kgv_hash_headers", "kgv_validate_headers_in_isolation"])
@pytest.mark.parametrize("side", ["h", "d"])
def test_header_arena_range_refused_on_either_side(ctx, oracle, call, side):
    """a header whose levels_off / parents_off range leaves the arena is refused, naming the call, whether the arrays are host or device
    memory (the kernels find it; the call reports it after its synchronise)"""
    from rusty_kaspa_b200.headers import HEADER_DTYPE
    make, _, _ = _builder(ctx, oracle, call)
    for field in ("levels_off", "parents_off"):
        c = make()
        h = np.frombuffer(c.arrays["headers"][0].tobytes(), dtype=HEADER_DTYPE).copy()
        h[3][field] = (len(c.arrays["level_len"][0]) // 4) if field == "levels_off" else len(c.arrays["parents32"][0]) // 32
        if field == "levels_off":
            h[3]["n_levels"] = max(int(h[3]["n_levels"]), 1)
        c.arrays["headers"] = (u8(h), "in")
        names = make_names(make)
        sides = {n: ("h" if n in SPEC[call].get("host", []) else side) for n in names}
        rc, _, _, _, err = run(ctx, c, sides)
        assert rc == KGV_ERR_ARG and call in err and "arena" in err, (field, side, rc, err)


# ---------------------------------------------------------------------------------------------
# host-only and device-only arguments of the calls without a full matrix here
# ---------------------------------------------------------------------------------------------
def _window():
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.replay import REPLAY_BLOCK_DTYPE
    g = simgen.FastDag(seed=5, n_keys=32, n_nonces=64, coinbase_maturity=3, mix=(0.5, 0.2, 0.15, 0.15), frac_invalid=0.1, coinbase_outputs=4)
    g.generate(12, 8)
    b, first, pov = g.take()
    C = g.C
    g.close()
    blocks = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
    blocks["first_tx"], blocks["n_txs"], blocks["pov_daa_score"], blocks["flags"] = first[:-1], np.diff(first), pov, 1
    return b, blocks, first.astype(np.uint32), C


def _dev_copy(obj, keep):
    """a device copy of a ctypes struct or numpy array"""
    import torch
    raw = bytes(obj) if isinstance(obj, ctypes.Structure) else np.ascontiguousarray(obj).tobytes()
    t = torch.frombuffer(bytearray(raw + b"\0" * 8), dtype=torch.uint8).cuda()
    keep.append(t)
    return t.data_ptr()


def _refusals(ctx, b, blocks, first, C, keep):
    """(call, argument, fn(ptr) -> rc, outputs to check untouched): ptr is a device pointer given for a host-only argument"""
    from rusty_kaspa_b200 import Params
    from rusty_kaspa_b200.replay import DagReplayer, RESULT_DTYPE
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    lib, h = ctx._lib, ctx._h
    params = Params(coinbase_maturity=3, storage_mass_parameter=C)
    rp = DagReplayer(ctx, params, 1 << 12)
    keep.append(rp)
    cb = _KgvTxBatch(b.txs.ctypes.data, len(b.txs), b.inputs.ctypes.data, len(b.inputs), b.outputs.ctypes.data, len(b.outputs), None,
                     b.arena.ctypes.data, len(b.arena))
    keep.append(cb)
    nt = len(b.txs)
    res = np.full(nt * RESULT_DTYPE.itemsize, SENTINEL, np.uint8)
    acc = np.full(nt, SENTINEL, np.uint8)
    big = np.full(1 << 16, SENTINEL, np.uint8)       # generic host output / struct stand-in
    prm = ctypes.byref(rp.tv.params)
    sz = ctypes.c_size_t(0)
    szp = ctypes.byref(sz)
    P = lambda p: ctypes.cast(p, ctypes.POINTER(ctypes.c_size_t))
    nb = len(blocks)
    return [
        ("kgv_validate_txs", "params", lambda p: lib.kgv_validate_txs(h, rp.us._h, ctypes.byref(cb), 10, 0, p, res.ctypes.data), [res]),
        ("kgv_validate_populated", "params", lambda p: lib.kgv_validate_populated(h, ctypes.byref(cb), 10, 0, p, res.ctypes.data), [res]),
        ("kgv_replay_window", "blocks", lambda p: lib.kgv_replay_window(h, rp.us._h, ctypes.byref(cb), p, nb, prm, res.ctypes.data, acc.ctypes.data, None),
         [res, acc]),
        ("kgv_replay_window", "params", lambda p: lib.kgv_replay_window(h, rp.us._h, ctypes.byref(cb), blocks.ctypes.data, nb, p, res.ctypes.data,
                                                                         acc.ctypes.data, None), [res, acc]),
        ("kgv_replay_window", "stats", lambda p: lib.kgv_replay_window(h, rp.us._h, ctypes.byref(cb), blocks.ctypes.data, nb, prm, res.ctypes.data,
                                                                        acc.ctypes.data, p), [res, acc]),
        ("kgv_validate_txs_in_isolation", "rules", lambda p: lib.kgv_validate_txs_in_isolation(h, ctypes.byref(cb), p, 0, 0, 0, res.ctypes.data, None),
         [res]),
        ("kgv_check_txs_standard_in_isolation", "policy",
         lambda p: lib.kgv_check_txs_standard_in_isolation(h, ctypes.byref(cb), p, big.ctypes.data, res.ctypes.data, None), [res]),
        ("kgv_check_txs_standard_in_context", "policy",
         lambda p: lib.kgv_check_txs_standard_in_context(h, ctypes.byref(cb), p, big.ctypes.data, big.ctypes.data, big.ctypes.data, res.ctypes.data,
                                                         None), [res]),
        ("kgv_validate_mempool_txs", "params",
         lambda p: lib.kgv_validate_mempool_txs(h, rp.us._h, ctypes.byref(cb), 10, p, None, res.ctypes.data, big.ctypes.data, None, None, 0, None),
         [res]),
        ("kgv_validate_mempool_txs", "scripts_used",
         lambda p: lib.kgv_validate_mempool_txs(h, rp.us._h, ctypes.byref(cb), 10, prm, None, res.ctypes.data, big.ctypes.data, None, None, 0, P(p)),
         [res]),
        ("kgv_validate_mempool_txs_in_parallel", "rules",
         lambda p: lib.kgv_validate_mempool_txs_in_parallel(h, rp.us._h, ctypes.byref(cb), 10, 0, prm, p, None, res.ctypes.data, big.ctypes.data,
                                                            None, None, None, 0, None), [res]),
        ("kgv_validate_mempool_txs_with_policy", "policy",
         lambda p: lib.kgv_validate_mempool_txs_with_policy(h, rp.us._h, ctypes.byref(cb), 10, 0, prm, big.ctypes.data, None, res.ctypes.data,
                                                            big.ctypes.data, None, None, None, 0, None, p, None), [res]),
        ("kgv_validate_block_bodies", "block_first_tx",
         lambda p: lib.kgv_validate_block_bodies(h, ctypes.byref(cb), p, 1, big.ctypes.data, big.ctypes.data, big.ctypes.data, 0, res.ctypes.data, None,
                                                 None), [res]),
        ("kgv_validate_block_bodies", "rules",
         lambda p: lib.kgv_validate_block_bodies(h, ctypes.byref(cb), first.ctypes.data, nb, big.ctypes.data, p, big.ctypes.data, 0, res.ctypes.data,
                                                 None, None), [res]),
        ("kgv_validate_block_bodies", "body_rules",
         lambda p: lib.kgv_validate_block_bodies(h, ctypes.byref(cb), first.ctypes.data, nb, big.ctypes.data, big.ctypes.data, p, 0, res.ctypes.data,
                                                 None, None), [res]),
        ("kgv_validate_headers_in_isolation", "rules",
         lambda p: lib.kgv_validate_headers_in_isolation(h, big.ctypes.data, 1, None, 0, None, 0, p, res.ctypes.data, None, None), [res]),
        ("kgv_merkle_roots", "first", lambda p: lib.kgv_merkle_roots(h, big.ctypes.data, p, 1, res.ctypes.data), [res]),
        ("kgv_block_hash_merkle_roots", "block_first_tx", lambda p: lib.kgv_block_hash_merkle_roots(h, ctypes.byref(cb), p, nb, res.ctypes.data), [res]),
        ("kgv_block_set_checks", "block_first_tx", lambda p: lib.kgv_block_set_checks(h, ctypes.byref(cb), p, nb, res.ctypes.data), [res]),
        ("kgv_utxo_import_chunk", "numerator384",
         lambda p: lib.kgv_utxo_import_chunk(h, rp.us._h, big.ctypes.data, big.ctypes.data, big.ctypes.data, 0, 1, p), []),
        ("kgv_utxo_export", "n_out", lambda p: lib.kgv_utxo_export(h, rp.us._h, big.ctypes.data, big.ctypes.data, big.ctypes.data, 1, 1, P(p), szp), [big]),
        ("kgv_utxo_export", "bytes_out", lambda p: lib.kgv_utxo_export(h, rp.us._h, big.ctypes.data, big.ctypes.data, big.ctypes.data, 1, 1, szp, P(p)),
         [big]),
    ]


def _host_struct_for(call, arg, rp, blocks, first):
    """the host value whose device copy is passed"""
    if arg in ("params",):
        return rp.tv.params
    if arg == "blocks":
        return blocks
    if arg in ("block_first_tx", "first"):
        return first
    return np.zeros(256, np.uint8)  # rules / policy / stats / counts / numerator: contents never read


@pytest.mark.gpu
def test_host_only_arguments_refused():
    """a device pointer for each host-only argument: KGV_ERR_ARG naming the call and the argument, outputs untouched, no launch"""
    import rusty_kaspa_b200 as rk
    b, blocks, first, C = _window()
    c = rk.GpuContext(0)
    keep = []
    lib, h = c._lib, c._h
    cases = _refusals(c, b, blocks, first, C, keep)
    rp = keep[0]
    seen = set()
    for call, arg, fn, outs in cases:
        assert arg in SPEC[call].get("host", []), (call, arg)
        seen.add((call, arg))
        snap = [o.copy() for o in outs]
        before = lib.kgv_launch_count(h)
        rc = fn(_dev_copy(_host_struct_for(call, arg, rp, blocks, first), keep))
        err = lib.kgv_last_error(h).decode()
        assert rc == KGV_ERR_ARG, (call, arg, rc, err)
        assert call in err and arg in err, (call, arg, err)
        assert lib.kgv_launch_count(h) == before, (call, arg)
        assert all((o == s).all() for o, s in zip(outs, snap)), (call, arg)
    rp.close()
    c.close()


@pytest.mark.gpu
def test_replay_follow_ups_refuse_device_host_arguments():
    """after a replay window: kgv_replay_muhash, kgv_replay_diffs and kgv_replay_verify_chain refuse device group offsets, rules and
    counts, and the refusals leave the window current (the host call still works)"""
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200 import Params
    from rusty_kaspa_b200.replay import DagReplayer, RESULT_DTYPE
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    b, blocks, first, C = _window()
    c = rk.GpuContext(0)
    lib, h = c._lib, c._h
    keep = []
    rp = DagReplayer(c, Params(coinbase_maturity=3, storage_mass_parameter=C), 1 << 12)
    cb = _KgvTxBatch(b.txs.ctypes.data, len(b.txs), b.inputs.ctypes.data, len(b.inputs), b.outputs.ctypes.data, len(b.outputs), None,
                     b.arena.ctypes.data, len(b.arena))
    nt, nb = len(b.txs), len(blocks)
    res = np.zeros(nt, dtype=RESULT_DTYPE)
    assert lib.kgv_replay_window(h, rp.us._h, ctypes.byref(cb), blocks.ctypes.data, nb, ctypes.byref(rp.tv.params), res.ctypes.data, None, None) == 0
    gf = np.array([0, nb], dtype=np.uint32)
    vals = np.full(768, SENTINEL, np.uint8)
    z = np.zeros(4096, np.uint8)
    sz = [ctypes.c_size_t(0) for _ in range(3)]
    P = lambda p: ctypes.cast(p, ctypes.POINTER(ctypes.c_size_t))
    cases = [
        ("kgv_replay_muhash", "group_first_block", lambda d: lib.kgv_replay_muhash(h, d, 1, vals.ctypes.data)),
        ("kgv_replay_diffs", "group_first_block", lambda d: lib.kgv_replay_diffs(h, d, 1, None, None, None, None, None, None, 0, 0, 0, *map(ctypes.byref, sz))),
        ("kgv_replay_diffs", "n_rem_out", lambda d: lib.kgv_replay_diffs(h, gf.ctypes.data, 1, None, None, None, None, None, None, 0, 0, 0, P(d),
                                                                          ctypes.byref(sz[1]), ctypes.byref(sz[2]))),
        ("kgv_replay_diffs", "n_add_out", lambda d: lib.kgv_replay_diffs(h, gf.ctypes.data, 1, None, None, None, None, None, None, 0, 0, 0,
                                                                          ctypes.byref(sz[0]), P(d), ctypes.byref(sz[2]))),
        ("kgv_replay_diffs", "bytes_out", lambda d: lib.kgv_replay_diffs(h, gf.ctypes.data, 1, None, None, None, None, None, None, 0, 0, 0,
                                                                          ctypes.byref(sz[0]), ctypes.byref(sz[1]), P(d))),
        ("kgv_replay_verify_chain", "body_rules",
         lambda d: lib.kgv_replay_verify_chain(h, gf.ctypes.data, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, d, vals.ctypes.data, None, None)),
        ("kgv_replay_verify_chain", "group_first_block",
         lambda d: lib.kgv_replay_verify_chain(h, d, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, vals.ctypes.data, None, None)),
        ("kgv_replay_verify_chain", "rules",
         lambda d: lib.kgv_replay_verify_chain(h, gf.ctypes.data, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, d, z.ctypes.data, vals.ctypes.data, None, None)),
    ]
    for call, arg, fn in cases:
        before = lib.kgv_launch_count(h)
        rc = fn(_dev_copy(gf if arg == "group_first_block" else z[:64], keep))
        err = lib.kgv_last_error(h).decode()
        assert rc == KGV_ERR_ARG and call in err and arg in err, (call, arg, rc, err)
        assert lib.kgv_launch_count(h) == before and (vals == SENTINEL).all(), (call, arg)
    # kgv_replay_diffs: device entry arrays 8-byte aligned (the others of the group aligned, one entry array off by 4)
    import torch
    dbuf = [torch.zeros(1 << 16, dtype=torch.uint8, device="cuda") for _ in range(6)]
    for bad in (1, 3):
        ptr = [t.data_ptr() for t in dbuf]
        ptr[bad] += 4
        before = lib.kgv_launch_count(h)
        rc = lib.kgv_replay_diffs(h, gf.ctypes.data, 1, ptr[0], ptr[2], ptr[1], ptr[4], ptr[3], ptr[5], 256, 256, 1 << 12, *map(ctypes.byref, sz))
        err = lib.kgv_last_error(h).decode()
        assert rc == KGV_ERR_ARG and "kgv_replay_diffs" in err and "aligned" in err, (bad, rc, err)
        assert lib.kgv_launch_count(h) == before
    assert lib.kgv_replay_muhash(h, gf.ctypes.data, 1, vals.ctypes.data) == 0, lib.kgv_last_error(h)
    rp.close()
    c.close()


@pytest.mark.gpu
def test_device_only_arguments_refused():
    """the kgv_comm.cu calls take device arrays only: a host array is refused naming the call, before anything is launched"""
    import torch
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200.comm import ShardComm
    c = rk.GpuContext(0)
    lib, h = c._lib, c._h
    comm = ShardComm(c, 1, 0, None, slice_capacity=1 << 12)
    host = np.zeros(64, np.uint8)
    dev = torch.zeros(64, dtype=torch.uint8, device="cuda")
    ep = ctypes.c_uint64(0)
    cases = [
        ("kgv_shard_publish_bitmap", lambda: lib.kgv_shard_publish_bitmap(h, comm._h, host.ctypes.data, 64, ctypes.byref(ep))),
        ("kgv_shard_publish_bytes", lambda: lib.kgv_shard_publish_bytes(h, comm._h, host.ctypes.data, 64, ctypes.byref(ep))),
        ("kgv_shard_wait", lambda: lib.kgv_shard_wait(h, comm._h, 0, 64, host.ctypes.data)),
        ("kgv_shard_allgather", lambda: lib.kgv_shard_allgather(h, comm._h, host.ctypes.data, 64, dev.data_ptr())),
        ("kgv_shard_allgather", lambda: lib.kgv_shard_allgather(h, comm._h, dev.data_ptr(), 64, host.ctypes.data)),
        ("kgv_shard_publish_bitmap", lambda: lib.kgv_shard_publish_bitmap(h, comm._h, dev.data_ptr(), 64,
                                                                          ctypes.cast(dev.data_ptr(), ctypes.POINTER(ctypes.c_uint64)))),
        ("kgv_shard_publish_bytes", lambda: lib.kgv_shard_publish_bytes(h, comm._h, dev.data_ptr(), 64,
                                                                        ctypes.cast(dev.data_ptr(), ctypes.POINTER(ctypes.c_uint64)))),
    ]
    for call, fn in cases:
        before = lib.kgv_launch_count(h)
        rc = fn()
        err = lib.kgv_last_error(h).decode()
        assert rc == KGV_ERR_ARG and call in err, (call, rc, err)
        assert lib.kgv_launch_count(h) == before, call
    comm.close()
    c.close()


# ---------------------------------------------------------------------------------------------
# value-dependent refusals, decided after staging, on either side
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("side", ["h", "d"])
def test_import_script_range_refused_on_either_side(ctx, side):
    """an entry whose script leaves the arena is refused whether entries (and keys36) are host or device memory, and whatever the side
    of the other array"""
    import rusty_kaspa_b200 as rk
    n = 8
    keys, ent, arena, n_bytes, _ = _utxo_chunk(n, 23, bad_script=True)
    for keys_side in "hd":
        us = rk.GpuUtxoSet(ctx, 1 << 10)
        num = np.frombuffer(_le(1), dtype=np.uint8).copy()
        keep = []
        pk, _ = _place(u8(keys), keys_side, 0, keep)
        pe, _ = _place(u8(ent), side, 0, keep)
        pb, _ = _place(arena, side, 0, keep)
        before = ctx._lib.kgv_launch_count(ctx._h)
        rc = ctx._lib.kgv_utxo_import_chunk(ctx._h, us._h, pk, pe, pb, n_bytes, n, num.ctypes.data)
        assert rc == KGV_ERR_ARG and "kgv_utxo_import_chunk" in ctx._lib.kgv_last_error(ctx._h).decode(), (side, keys_side, rc)
        assert ctx._lib.kgv_launch_count(ctx._h) == before
        assert num.tobytes() == _le(1)
        cnt = ctypes.c_uint64(0)
        assert ctx._lib.kgv_utxo_count(ctx._h, us._h, ctypes.byref(cnt)) == 0 and cnt.value == 0
        us.close()


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["h", "d"])
def test_check_scripts_index_range_refused_on_either_side(ctx, side):
    """kgv_check_scripts refuses a transaction index >= n_txs whether tx_indices is host or device memory"""
    from rusty_kaspa_b200.validator import RESULT_DTYPE
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    b, _, _, _ = _window()
    ent = np.zeros(max(len(b.inputs), 1) * 32, np.uint8)
    cb = _KgvTxBatch(b.txs.ctypes.data, len(b.txs), b.inputs.ctypes.data, len(b.inputs), b.outputs.ctypes.data, len(b.outputs), ent.ctypes.data,
                     b.arena.ctypes.data, len(b.arena))
    idx = np.array([0, len(b.txs)], dtype=np.uint32)
    keep = []
    pi, _ = _place(u8(idx), side, 0, keep)
    res = np.full(2 * RESULT_DTYPE.itemsize, SENTINEL, np.uint8)
    before = ctx._lib.kgv_launch_count(ctx._h)
    rc = ctx._lib.kgv_check_scripts(ctx._h, ctypes.byref(cb), pi, 2, res.ctypes.data)
    assert rc == KGV_ERR_ARG and "kgv_check_scripts" in ctx._lib.kgv_last_error(ctx._h).decode(), (side, rc)
    assert ctx._lib.kgv_launch_count(ctx._h) == before and (res == SENTINEL).all()


# ---------------------------------------------------------------------------------------------
# staging reuse: d_io grows, parks and is reused across calls of one context
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_staging_reuse_matches_fresh_contexts():
    """host-array calls at growing, shrinking and growing sizes on one context, device-only calls and kgv_synchronize in between, and an
    import (whose inner kgv_muhash_combine stages into the same d_io offsets) after a larger call: every result equals the same call on
    a fresh context, and the imported table's digest and multiset equal the reference's"""
    import torch
    import rusty_kaspa_b200 as rk
    pr = _pyref()
    one = rk.GpuContext(0)

    def elements(c, n, seed):
        make, anchor = _muhash_elements(c, n, seed)
        r = run(c, make(), {})
        anchor(r[2], b"")
        return r[:3]

    def device_combine(c, seed):
        rnd = random.Random(seed)
        vals = [_rand_residue(rnd) for _ in range(4)]
        t = [torch.from_numpy(np.frombuffer(_le(v), dtype=np.uint8).copy()).cuda() for v in vals]
        assert c._lib.kgv_muhash_combine(c._h, *[x.data_ptr() for x in t]) == 0
        assert c._lib.kgv_synchronize(c._h) == 0
        return t[0].cpu().numpy().tobytes() + t[1].cpu().numpy().tobytes()

    def imported(c, n, seed):
        make, anchor = _utxo_import_chunk(c, n, seed)
        case = make()
        r = run(c, case, {})
        case.close()
        anchor(r[2], r[3])
        return r[:4]

    seq = [("e", 16, 31), ("e", 400, 32), ("c", 0, 33), ("e", 5, 34), ("i", 12, 35), ("e", 900, 36), ("c", 0, 37), ("i", 3, 38), ("e", 2, 39),
           ("i", 200, 40)]
    for kind, n, seed in seq:
        got = {"e": elements, "c": lambda c, n, s: device_combine(c, s), "i": imported}[kind](one, n, seed)
        fresh = rk.GpuContext(0)
        want = {"e": elements, "c": lambda c, n, s: device_combine(c, s), "i": imported}[kind](fresh, n, seed)
        fresh.close()
        assert got == want, (kind, n, seed)
    # one table fed chunk by chunk on the reused context: its digest equals a single import on a fresh context, its multiset the reference's
    keys, ent, arena, n_bytes, scripts = _utxo_chunk(30, 41)
    us = rk.GpuUtxoSet(one, 1 << 10)
    num = np.frombuffer(_le(1), dtype=np.uint8).copy()
    for lo, hi in ((0, 20), (20, 30)):
        k, e = keys[lo:hi].copy(), ent[lo:hi].copy()
        assert one._lib.kgv_utxo_import_chunk(one._h, us._h, k.ctypes.data, e.ctypes.data, arena.ctypes.data, n_bytes, hi - lo,
                                              num.ctypes.data) == 0, one._lib.kgv_last_error(one._h)
        elements(one, 600, 42 + lo)  # a larger host call in between
    fresh = rk.GpuContext(0)
    us2 = rk.GpuUtxoSet(fresh, 1 << 10)
    num2 = np.frombuffer(_le(1), dtype=np.uint8).copy()
    assert fresh._lib.kgv_utxo_import_chunk(fresh._h, us2._h, keys.ctypes.data, ent.ctypes.data, arena.ctypes.data, n_bytes, 30, num2.ctypes.data) == 0
    assert us.digest() == us2.digest() == _oracle_digest(keys, ent, scripts)
    m = pr.MuHash()
    for i in range(30):
        x = ent[i]
        m.add_element(pr.utxo_element_bytes(keys[i, :32].tobytes(), int.from_bytes(keys[i, 32:].tobytes(), "little"), int(x["block_daa_score"]),
                                            int(x["amount"]), int(x["is_coinbase"]), int(x["spk_version"]), scripts[i]))
    assert num.tobytes() == num2.tobytes() == _le(m.num)
    us2.close()
    fresh.close()
    us.close()
    one.close()


def _oracle_digest(keys, ent, scripts):
    """the UTXO-set digest of ok_state_digest: sum mod 2^256 of the MuHashElement hashes of the entries, little-endian"""
    pr = _pyref()
    acc = 0
    for i in range(len(ent)):
        e = ent[i]
        data = pr.utxo_element_bytes(keys[i, :32].tobytes(), int.from_bytes(keys[i, 32:].tobytes(), "little"), int(e["block_daa_score"]),
                                     int(e["amount"]), int(e["is_coinbase"]), int(e["spk_version"]), scripts[i])
        acc = (acc + int.from_bytes(pr.blake2b_keyed(b"MuHashElement", data), "little")) % (1 << 256)
    return acc.to_bytes(32, "little")


@pytest.mark.gpu
def test_scalar_results_are_host_only(ctx):
    """kgv_utxo_count, kgv_utxo_digest, kgv_utxo_stats and kgv_sigcache_counters write their results on the host: a device pointer is
    refused, naming the call and the argument, before anything is launched"""
    import torch
    import rusty_kaspa_b200 as rk
    from rusty_kaspa_b200.validator import SigCache
    lib, h = ctx._lib, ctx._h
    us = rk.GpuUtxoSet(ctx, 1 << 10)
    sc = SigCache(ctx, 1024)
    dev = torch.full((256,), SENTINEL, dtype=torch.uint8, device="cuda")
    d = dev.data_ptr()
    u64 = lambda p: ctypes.cast(p, ctypes.POINTER(ctypes.c_uint64))
    host = [ctypes.c_uint64(0) for _ in range(4)]
    hp = [ctypes.byref(x) for x in host]
    cases = [("kgv_utxo_count", "count", lambda: lib.kgv_utxo_count(h, us._h, u64(d))),
             ("kgv_utxo_digest", "out32", lambda: lib.kgv_utxo_digest(h, us._h, d)),
             ("kgv_utxo_stats", "out", lambda: lib.kgv_utxo_stats(h, us._h, d))]
    for k, arg in enumerate(("hits", "inserts", "lookups", "evictions")):
        ps = list(hp)
        ps[k] = u64(d)
        cases.append(("kgv_sigcache_counters", arg, lambda ps=ps: lib.kgv_sigcache_counters(h, sc._h, *ps)))
    for call, arg, fn in cases:
        assert arg in SPEC[call]["host"]
        before = lib.kgv_launch_count(h)
        rc = fn()
        err = lib.kgv_last_error(h).decode()
        assert rc == KGV_ERR_ARG and call in err and arg in err, (call, arg, rc, err)
        assert lib.kgv_launch_count(h) == before, call
    assert lib.kgv_synchronize(h) == 0
    assert (dev.cpu().numpy() == SENTINEL).all()
    sc.close()
    us.close()


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["h", "d"])
def test_replay_block_tiling_refused_on_either_side(ctx, side):
    """blocks that do not tile the batch are refused whether the batch is host or device memory (blocks are host memory by contract)"""
    from rusty_kaspa_b200 import Params
    from rusty_kaspa_b200.replay import DagReplayer
    from rusty_kaspa_b200.validator import RESULT_DTYPE
    b, blocks, _, C = _window()
    rp = DagReplayer(ctx, Params(coinbase_maturity=3, storage_mass_parameter=C), 1 << 12)
    keep, p = [], {}
    for name, (data, _) in _batch_arrays(b).items():
        p[name], _ = _place(data, side, 0, keep)
    cb = _c_batch(b, p)
    res = np.full(len(b.txs) * RESULT_DTYPE.itemsize, SENTINEL, np.uint8)
    for how in ("gap", "short", "flags"):
        bad = blocks.copy()
        if how == "gap":
            bad["first_tx"][2] += 1
        elif how == "short":
            bad["n_txs"][-1] -= 1
        else:
            bad["flags"][1] = 8
        before = ctx._lib.kgv_launch_count(ctx._h)
        rc = ctx._lib.kgv_replay_window(ctx._h, rp.us._h, ctypes.byref(cb), bad.ctypes.data, len(bad), ctypes.byref(rp.tv.params), res.ctypes.data,
                                        None, None)
        err = ctx._lib.kgv_last_error(ctx._h).decode()
        assert rc == KGV_ERR_ARG and "kgv_replay_window" in err and "replay blocks" in err, (how, side, rc, err)
        assert ctx._lib.kgv_launch_count(ctx._h) == before and (res == SENTINEL).all()
    rp.close()
