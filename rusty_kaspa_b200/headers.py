"""Host-side Python mirror of header validation in isolation (include/kgv.h: kgv_hash_headers, kgv_validate_headers_in_isolation).

`HeaderBatch` packs header dicts (blocks_json.header_from_json) into the C records: one HEADER_DTYPE per header and an arena of the
expanded parents_by_level (level sizes + parent hashes).  `hash_headers` returns the block hashes and pre-PoW hashes;
`validate_headers_in_isolation` returns HeaderProcessor::validate_header_in_isolation's verdict, the block level and the pass bit of the
proof of work for every header (consensus/src/pipeline/header_processor/pre_ghostdag_validation.rs:17-24).
"""
import ctypes

import numpy as np

from .verifier import _addr_and_keepalive

HEADER_DTYPE = np.dtype([("hash_merkle_root", "u1", 32), ("accepted_id_merkle_root", "u1", 32), ("utxo_commitment", "u1", 32),
                         ("pruning_point", "u1", 32), ("blue_work", "u1", 24), ("timestamp", "<u8"), ("nonce", "<u8"), ("daa_score", "<u8"),
                         ("blue_score", "<u8"), ("parents_off", "<u8"), ("levels_off", "<u4"), ("n_levels", "<u4"), ("bits", "<u4"),
                         ("version", "<u2"), ("pad_", "<u2")])
assert HEADER_DTYPE.itemsize == 208
HEADER_RESULT_DTYPE = np.dtype([("status", "<u4"), ("level", "u1"), ("pow_passed", "u1"), ("pad_", "<u2"), ("a", "<u8"), ("b", "<u8")])
assert HEADER_RESULT_DTYPE.itemsize == 24
# KGV_HEADER_* (include/kgv.h): the RuleError of validate_header_in_isolation each status stands for
HEADER_STATUS = {"Ok": 0, "WrongBlockVersion": 1, "TimeTooFarIntoTheFuture": 2, "NoParents": 3, "TooManyParents": 4, "OriginParent": 5, "InvalidPoW": 6}
SKIP_POW = 1


class HeaderRules(ctypes.Structure):
    """kgv_header_rules.  The defaults are mainnet's (constants::BLOCK_VERSION, MAINNET_PARAMS: max_block_parents of the 10 BPS blockrate,
    max_block_level 225, TIMESTAMP_DEVIATION_TOLERANCE 132 s); now_ms stands for the reference's unix_now() and defaults to 0."""
    _fields_ = [("timestamp_deviation_tolerance", ctypes.c_uint64), ("now_ms", ctypes.c_uint64), ("block_version", ctypes.c_uint32),
                ("max_block_parents", ctypes.c_uint32), ("max_block_level", ctypes.c_uint32), ("flags", ctypes.c_uint32)]

    def __init__(self, timestamp_deviation_tolerance=132, now_ms=0, block_version=1, max_block_parents=16, max_block_level=225, skip_pow=False):
        super().__init__(timestamp_deviation_tolerance, now_ms, block_version, max_block_parents, max_block_level, SKIP_POW if skip_pow else 0)


class HeaderBatch:
    """headers: HEADER_DTYPE[n]; level_len: uint32 level sizes; parents: (m, 32) uint8 parent hashes.  Header k's levels are
    level_len[levels_off : levels_off + n_levels] and its parents start at parents[parents_off]."""

    def __init__(self, headers, level_len, parents):
        self.headers = np.ascontiguousarray(headers, dtype=HEADER_DTYPE)
        self.level_len = np.ascontiguousarray(level_len, dtype=np.uint32)
        self.parents = np.ascontiguousarray(parents, dtype=np.uint8).reshape(-1, 32)

    def __len__(self):
        return len(self.headers)

    @classmethod
    def from_dicts(cls, hs):
        """header dicts with version, parents_by_level (expanded), the three roots, timestamp, bits, nonce, daa_score, blue_score,
        blue_work (int) and pruning_point."""
        arr = np.zeros(len(hs), dtype=HEADER_DTYPE)
        lens, pars = [], []
        for k, h in enumerate(hs):
            r = arr[k]
            for f in ("hash_merkle_root", "accepted_id_merkle_root", "utxo_commitment", "pruning_point"):
                r[f] = np.frombuffer(h[f], dtype=np.uint8)
            r["blue_work"] = np.frombuffer(int(h["blue_work"]).to_bytes(24, "big"), dtype=np.uint8)
            for f in ("timestamp", "nonce", "daa_score", "blue_score", "bits", "version"):
                r[f] = h[f]
            r["parents_off"], r["levels_off"], r["n_levels"] = len(pars), len(lens), len(h["parents_by_level"])
            for lvl in h["parents_by_level"]:
                lens.append(len(lvl))
                pars.extend(lvl)
        parents = np.frombuffer(b"".join(pars), dtype=np.uint8).reshape(-1, 32) if pars else np.zeros((0, 32), dtype=np.uint8)
        return cls(arr, np.array(lens, dtype=np.uint32), parents)


def _args(ctx, batch):
    keep = []
    addr = []
    for buf in (batch.headers, batch.parents, batch.level_len):
        a, _, k = _addr_and_keepalive(buf, 0)
        addr.append(a if buf.size else None)
        keep.append(k)
    return addr, keep


def hash_headers(ctx, batch, want_pre_pow=True):
    """kgv_hash_headers: (block hashes, pre-PoW hashes or None), each (n, 32) uint8."""
    n = len(batch)
    hashes = np.zeros((max(n, 1), 32), dtype=np.uint8)
    pre = np.zeros((max(n, 1), 32), dtype=np.uint8) if want_pre_pow else None
    (ah, ap, al), _keep = _args(ctx, batch)
    ctx._check(ctx._lib.kgv_hash_headers(ctx._h, ah, n, ap, len(batch.parents), al, len(batch.level_len), hashes.ctypes.data,
                                         pre.ctypes.data if pre is not None else None))
    return hashes[:n], (pre[:n] if pre is not None else None)


def validate_headers_in_isolation(ctx, batch, rules=None, want_hash=False, want_pow=False):
    """kgv_validate_headers_in_isolation: HEADER_RESULT_DTYPE[n], plus the block hashes and the PoW values ((n, 32) uint8, the value
    little-endian) when asked for (else None)."""
    rules = rules or HeaderRules()
    n = len(batch)
    res = np.zeros(max(n, 1), dtype=HEADER_RESULT_DTYPE)
    hashes = np.zeros((max(n, 1), 32), dtype=np.uint8) if want_hash else None
    pw = np.zeros((max(n, 1), 32), dtype=np.uint8) if want_pow else None
    (ah, ap, al), _keep = _args(ctx, batch)
    ctx._check(ctx._lib.kgv_validate_headers_in_isolation(ctx._h, ah, n, ap, len(batch.parents), al, len(batch.level_len), ctypes.byref(rules),
                                                          res.ctypes.data, hashes.ctypes.data if hashes is not None else None,
                                                          pw.ctypes.data if pw is not None else None))
    return res[:n], (hashes[:n] if hashes is not None else None), (pw[:n] if pw is not None else None)


def debug_pow_matrix(ctx, op, data, n):
    """kgv_debug_pow_matrix: op 0 ranks n u16 matrices (n, 64, 64) -> uint32[n]; op 1 generates from n 32-byte seeds ->
    ((n, 64, 64) uint8 matrices, uint32[n] matrices drawn)."""
    src = np.ascontiguousarray(data)
    out = np.zeros(n * (4 if op == 0 else 4100), dtype=np.uint8)
    ctx._check(ctx._lib.kgv_debug_pow_matrix(ctx._h, op, src.ctypes.data, n, out.ctypes.data))
    if op == 0:
        return out.view(np.uint32)
    rec = out.reshape(n, 4100)
    return rec[:, :4096].reshape(n, 64, 64).copy(), rec[:, 4096:].copy().view(np.uint32).reshape(n)
