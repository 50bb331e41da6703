"""ctypes loader for libkgv.so (the C-ABI drop-in boundary, include/kgv.h).

There is deliberately no fallback: if the CUDA library is missing or no device is usable the
import of a context fails loudly.  Nothing under oracle/ is ever touched from here.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# KGV_LIB lets the tuning scripts in tools/ point at an alternative build of the same CUDA library
LIB_PATH = os.environ.get("KGV_LIB", os.path.join(_HERE, "libkgv.so"))

KGV_OK = 0
SIG_INVALID, SIG_VALID, SIG_PK_PARSE_ERR, SIG_SIG_PARSE_ERR = 0, 1, 2, 3

# every symbol include/kgv.h declares: (name, restype, argtypes)
_c = ctypes
_u8p = _c.c_void_p  # raw addresses (host or device)
SYMBOLS = [
    ("kgv_create", _c.c_int, [_c.c_int, _c.c_uint32, _c.POINTER(_c.c_void_p)]),
    ("kgv_destroy", None, [_c.c_void_p]),
    ("kgv_set_stream", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_reset_stream", _c.c_int, [_c.c_void_p]),
    ("kgv_synchronize", _c.c_int, [_c.c_void_p]),
    ("kgv_last_error", _c.c_char_p, [_c.c_void_p]),
    ("kgv_launch_count", _c.c_uint64, [_c.c_void_p]),
    ("kgv_schnorr_verify", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_ecdsa_verify", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_status_to_bitmap", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_tx_ids", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p]),
    ("kgv_tx_hashes", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p]),
    ("kgv_sighash", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_validate_populated", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_uint32, _c.c_void_p, _u8p]),
    ("kgv_utxo_create", _c.c_int, [_c.c_void_p, _c.c_uint64, _c.POINTER(_c.c_void_p)]),
    ("kgv_utxo_destroy", None, [_c.c_void_p, _c.c_void_p]),
    ("kgv_utxo_view_create", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint64, _c.POINTER(_c.c_void_p)]),
    ("kgv_utxo_view_commit", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_utxo_view_discard", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_utxo_stats", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p]),
    ("kgv_utxo_rehash", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint64]),
    ("kgv_utxo_set_max_load", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint32]),
    ("kgv_utxo_lookup", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p, _u8p, _c.c_uint32, _u8p]),
    ("kgv_utxo_apply_diff", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p, _u8p, _u8p, _u8p, _c.c_size_t, _c.c_size_t, _u8p]),
    ("kgv_utxo_count", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_uint64)]),
    ("kgv_utxo_digest", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p]),
    ("kgv_batch_prefetch", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_utxo_export", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_size_t, _c.POINTER(_c.c_size_t), _c.POINTER(_c.c_size_t)]),
    ("kgv_utxo_import_chunk", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_size_t, _c.c_void_p]),
    ("kgv_validate_txs", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_uint32, _c.c_void_p, _u8p]),
    ("kgv_utxo_apply_accepted", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _u8p, _c.c_uint64]),
    ("kgv_validate_mempool_txs", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_void_p, _u8p, _u8p, _u8p, _u8p, _u8p, _c.c_size_t,
                                            _c.POINTER(_c.c_size_t)]),
    ("kgv_validate_txs_in_isolation", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_uint64, _c.c_uint32, _u8p, _u8p]),
    ("kgv_validate_mempool_txs_in_parallel", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_uint64, _c.c_void_p, _c.c_void_p, _u8p, _u8p,
                                                        _u8p, _u8p, _u8p, _u8p, _c.c_size_t, _c.POINTER(_c.c_size_t)]),
    ("kgv_check_txs_standard_in_isolation", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _u8p, _u8p, _u8p]),
    ("kgv_check_txs_standard_in_context", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _u8p, _u8p, _u8p, _u8p, _u8p]),
    ("kgv_outputs_dust", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint64, _u8p]),
    ("kgv_validate_mempool_txs_with_policy", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_uint64, _c.c_void_p, _c.c_void_p, _u8p, _u8p,
                                                        _u8p, _u8p, _u8p, _u8p, _c.c_size_t, _c.POINTER(_c.c_size_t), _c.c_void_p, _u8p]),
    ("kgv_sigcache_create", _c.c_int, [_c.c_void_p, _c.c_uint64, _c.POINTER(_c.c_void_p)]),
    ("kgv_sigcache_destroy", None, [_c.c_void_p]),
    ("kgv_sigcache_clear", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_sigcache_counters", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_uint64), _c.POINTER(_c.c_uint64), _c.POINTER(_c.c_uint64), _c.POINTER(_c.c_uint64)]),
    ("kgv_set_sigcache", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_keycache_create", _c.c_int, [_c.c_void_p, _c.c_uint64, _c.c_uint64]),
    ("kgv_keycache_share", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_keycache_destroy", _c.c_int, [_c.c_void_p]),
    ("kgv_keycache_clear", _c.c_int, [_c.c_void_p]),
    ("kgv_keycache_counter", _c.c_uint64, [_c.c_void_p, _c.c_int, _c.c_int]),
    ("kgv_set_keycache", _c.c_int, [_c.c_void_p, _c.c_int]),
    ("kgv_comm_unique_id", _c.c_int, [_u8p]),
    ("kgv_comm_create", _c.c_int, [_c.c_void_p, _c.c_int, _c.c_int, _u8p, _c.c_size_t, _c.POINTER(_c.c_void_p)]),
    ("kgv_comm_destroy", None, [_c.c_void_p]),
    ("kgv_comm_export", _c.c_int, [_c.c_void_p, _u8p]),
    ("kgv_comm_import", _c.c_int, [_c.c_void_p, _u8p]),
    ("kgv_comm_connect_local", _c.c_int, [_c.POINTER(_c.c_void_p), _c.c_int]),
    ("kgv_shard_allgather", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_shard_publish_bitmap", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _c.POINTER(_c.c_uint64)]),
    ("kgv_shard_publish_bytes", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _c.POINTER(_c.c_uint64)]),
    ("kgv_shard_wait", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_uint64, _c.c_size_t, _u8p]),
    ("kgv_set_sharding", _c.c_int, [_c.c_void_p, _c.c_void_p]),
    ("kgv_replay_window", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _c.c_void_p, _u8p, _u8p, _c.c_void_p]),
    ("kgv_merkle_roots", _c.c_int, [_c.c_void_p, _u8p, _u8p, _c.c_uint32, _u8p]),
    ("kgv_block_hash_merkle_roots", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_uint32, _u8p]),
    ("kgv_block_set_checks", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_uint32, _u8p]),
    ("kgv_validate_block_bodies", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_uint32, _u8p, _c.c_void_p, _c.c_void_p, _c.c_uint32, _u8p, _u8p, _u8p]),
    ("kgv_muhash_elements", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _c.c_size_t, _u8p, _u8p]),
    ("kgv_muhash_txs", _c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _u8p, _c.c_uint64, _u8p, _u8p]),
    ("kgv_muhash_combine", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _u8p]),
    ("kgv_muhash_finalize", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _u8p]),
    ("kgv_muhash_finalize_batch", _c.c_int, [_c.c_void_p, _u8p, _u8p, _c.c_size_t, _c.c_size_t, _u8p, _u8p]),
    ("kgv_muhash_prefix_combine", _c.c_int, [_c.c_void_p, _u8p, _u8p, _c.c_size_t]),
    ("kgv_replay_muhash", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_replay_diffs", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p, _u8p, _u8p, _u8p, _u8p, _u8p, _c.c_size_t, _c.c_size_t, _c.c_size_t,
                                    _c.POINTER(_c.c_size_t), _c.POINTER(_c.c_size_t), _c.POINTER(_c.c_size_t)]),
    ("kgv_replay_verify_chain", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p, _u8p, _u8p, _c.c_void_p, _c.c_void_p, _u8p, _u8p, _u8p]),
    ("kgv_utxo_muhash", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p]),
    ("kgv_hash_headers", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p, _c.c_size_t, _u8p, _c.c_size_t, _u8p, _u8p]),
    ("kgv_validate_headers_in_isolation", _c.c_int, [_c.c_void_p, _u8p, _c.c_size_t, _u8p, _c.c_size_t, _u8p, _c.c_size_t, _c.c_void_p, _u8p, _u8p, _u8p]),
    ("kgv_script_execute", _c.c_int, [_c.c_void_p, _c.c_uint32, _c.c_uint32, _c.c_void_p, _c.c_void_p, _u8p]),
    ("kgv_check_scripts_host", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_check_scripts", _c.c_int, [_c.c_void_p, _c.c_void_p, _u8p, _c.c_size_t, _u8p]),
    ("kgv_utxo_rows_encode", _c.c_int, [_u8p, _u8p, _u8p, _c.c_size_t, _c.c_size_t, _u8p, _u8p, _u8p, _u8p, _c.c_size_t, _c.c_size_t]),
    ("kgv_utxo_rows_decode", _c.c_int, [_u8p, _u8p, _u8p, _u8p, _c.c_size_t, _u8p, _u8p, _u8p, _c.c_size_t, _c.POINTER(_c.c_size_t)]),
    ("kgv_gtable_entry", _c.c_int, [_c.c_void_p, _c.c_int, _c.c_uint32, _u8p]),
    ("kgv_debug_selftest", _c.c_int, [_c.c_void_p, _c.c_int, _u8p, _u8p, _c.c_size_t]),
    ("kgv_debug_u3072_level", _c.c_int, [_c.c_void_p, _c.c_int, _u8p, _c.c_size_t, _u8p]),
    ("kgv_debug_pow_matrix", _c.c_int, [_c.c_void_p, _c.c_int, _u8p, _c.c_size_t, _u8p]),
    ("kgv_debug_schnorr_trace", _c.c_int, [_c.c_void_p, _u8p, _u8p, _u8p, _u8p, _u8p]),
    ("kgv_debug_key_form", _c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p]),
    ("kgv_debug_script_rounds", _c.c_int, [_c.c_void_p, _c.POINTER(_c.c_uint32)]),
]
TRACE_STAGES = 32
KEY_FORMS = ("no-cache", "inline", "plain", "comb")  # KGV_KEY_FORM_* in include/kgv.h


class KeyFormInfo(_c.Structure):
    _fields_ = [("n_items", _c.c_uint64), ("threads", _c.c_uint64), ("distinct_keys", _c.c_uint32), ("form", _c.c_int32)]

_lib = None


class KgvError(RuntimeError):
    pass


def load():
    """Loads libkgv.so (built by __graft_entry__.build()). Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KgvError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the ABI lost a symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
