"""The residency spec of tests/test_gpu_residency.py stays complete: every C entry point of include/kgv.h that takes a data pointer is in
it or is exempted here with a reason, and its call names are those of the table above class kgv_io (kgv_internal.h)."""
import os
import re

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# entry points with data pointers that have no side matrix, and why
EXEMPT = {
    "kgv_create": "returns the context handle into a host variable",
    "kgv_utxo_create": "returns a table handle into a host variable",
    "kgv_utxo_view_create": "returns a view handle into a host variable",
    "kgv_sigcache_create": "returns a cache handle into a host variable",
    "kgv_comm_create": "returns a communicator handle; the NCCL id is a host value",
    "kgv_comm_unique_id": "host-side NCCL id, no context",
    "kgv_comm_export": "host-side IPC handle of the communicator",
    "kgv_comm_import": "host-side IPC handles of the peers",
    "kgv_comm_connect_local": "an array of communicator handles",
    "kgv_set_stream": "takes a CUDA stream handle, not data",
    "kgv_batch_prefetch": "uploads a host batch ahead of a call; a device batch is a no-op",
    "kgv_script_execute": "host script engine, no device work",
    "kgv_check_scripts_host": "host script engine over a host batch",
    "kgv_utxo_rows_encode": "host row encoding, no context",
    "kgv_utxo_rows_decode": "host row decoding, no context",
    "kgv_gtable_entry": "debug hook: one table entry into a host array",
    "kgv_debug_schnorr_trace": "debug hook with host pointers only",
    "kgv_debug_key_form": "debug hook: a host struct",
    "kgv_debug_script_rounds": "debug hook: a host scalar",
    "kgv_debug_selftest": "debug hook with host pointers only",
    "kgv_debug_u3072_level": "debug hook with host pointers only (refuses device ones)",
    "kgv_debug_pow_matrix": "debug hook with host pointers only (refuses device ones)",
}
# handles are not data: a call whose only pointers are these takes no caller array
HANDLES = ("kgv_ctx", "kgv_utxo_table", "kgv_sigcache", "kgv_comm")


def _declarations():
    src = open(os.path.join(ROOT, "include", "kgv.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\bint\s+(kgv_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S):
        out[m.group(1)] = [p.strip() for p in m.group(2).split(",")]
    return out


def _takes_data_pointer(params):
    for p in params:
        if "*" not in p and "[" not in p:
            continue
        base = re.sub(r"\b(const|struct)\b", "", p).split("*")[0].split("[")[0].strip().split()
        if not base or base[0] not in HANDLES or p.count("*") > 1:
            return True
    return False


def _table_calls():
    src = open(os.path.join(ROOT, "rusty_kaspa_b200", "csrc", "kgv_internal.h")).read()
    start = src.index("// Which arrays of a call must share a side")
    end = src.index("// The arrays of a transaction batch are staged by kgv_batch_to_device")
    names = set()
    decls = _declarations()
    for line in src[start:end].splitlines():
        if not line.startswith("//   ") or line.startswith("//    "):
            continue  # not a row, or a continuation of the description column
        head = re.split(r"\s{2,}", line[5:])[0]  # the call column of the table
        if head.startswith("the kgv_comm.cu calls"):
            head = ""
        for m in re.finditer(r"(kgv_\w+)(\*?)((?:\s*/\s*_\w+)*)", head):
            name, star, rest = m.groups()
            if star:
                names |= {d for d in decls if d.startswith(name)}
            else:
                names.add(name)
            for suffix in re.findall(r"_\w+", rest):
                names.add(name.rsplit("_", 1)[0] + suffix)
        if "the kgv_comm.cu calls" in line:
            names |= {"kgv_shard_allgather", "kgv_shard_publish_bitmap", "kgv_shard_publish_bytes", "kgv_shard_wait"}
    return names


def _spec():
    import test_gpu_residency as R
    return R.SPEC


def test_every_data_entry_point_is_in_the_spec():
    spec = _spec()
    decls = _declarations()
    assert len(decls) > 60
    missing = [n for n, ps in decls.items() if _takes_data_pointer(ps) and n not in spec and n not in EXEMPT]
    assert not missing, "entry points with data pointers missing from SPEC in tests/test_gpu_residency.py: %s" % missing
    assert not set(spec) & set(EXEMPT)
    assert set(spec) <= set(decls), sorted(set(spec) - set(decls))
    assert set(EXEMPT) <= set(decls), sorted(set(EXEMPT) - set(decls))


def test_every_spec_call_has_a_matrix_or_a_reason():
    """a call of SPEC runs the side matrix (BUILDERS) or says what covers it instead (NO_MATRIX)"""
    import test_gpu_residency as R
    spec, built, reasons = set(R.SPEC), set(R.BUILDERS), R.NO_MATRIX
    assert not built & set(reasons), sorted(built & set(reasons))
    missing = sorted(spec - built - set(reasons))
    assert not missing, "calls of SPEC with neither a builder nor a reason: %s" % missing
    assert (built | set(reasons)) <= spec, sorted((built | set(reasons)) - spec)
    assert all(isinstance(r, str) and len(r) > 20 for r in reasons.values())


@pytest.mark.parametrize("call", ["kgv_utxo_lookup", "kgv_replay_diffs"])
def test_a_call_without_matrix_or_reason_is_named(call, monkeypatch):
    import test_gpu_residency as R
    monkeypatch.setattr(R, "BUILDERS", [c for c in R.BUILDERS if c != call])
    monkeypatch.setattr(R, "NO_MATRIX", {k: v for k, v in R.NO_MATRIX.items() if k != call})
    with pytest.raises(AssertionError, match=call):
        test_every_spec_call_has_a_matrix_or_a_reason()


def test_spec_names_match_the_kgv_io_table():
    table = _table_calls()
    spec = set(_spec())
    assert spec == table, ("in SPEC only: %s" % sorted(spec - table), "in the kgv_internal.h table only: %s" % sorted(table - spec))


def test_spec_arguments_are_parameters_of_the_call():
    """every argument the spec names is a parameter of the declaration ("batch" stands for the kgv_tx_batch)"""
    decls = _declarations()
    for call, s in _spec().items():
        params = {re.split(r"[\s*]+", p.split("[")[0].strip())[-1] for p in decls[call]}
        names = [n for g in s.get("together", []) for n in g] + s.get("own", []) + s.get("host", []) + s.get("device", []) + list(s.get("align", {}))
        for n in names:
            assert n in params or (n == "batch" and "batch" in params), (call, n, sorted(params))
        flat = [n for g in s.get("together", []) for n in g] + s.get("own", []) + s.get("host", []) + s.get("device", [])
        assert len(flat) == len(set(flat)), (call, "an argument listed twice")


@pytest.mark.parametrize("call", ["kgv_muhash_combine", "kgv_replay_window"])
def test_a_call_removed_from_the_spec_is_named(call, monkeypatch):
    """the completeness check names the call that is missing"""
    import test_gpu_residency as R
    monkeypatch.delitem(R.SPEC, call)
    with pytest.raises(AssertionError, match=call):
        test_every_data_entry_point_is_in_the_spec()
