"""Host-side Python mirror of the signature-verification boundary.

`GpuContext` owns a kgv_ctx (one per device).  `verify_schnorr_batch` / `verify_ecdsa_batch` are the
batch equivalents of the reference's per-signature `check_schnorr_signature` / `check_ecdsa_signature`
(crypto/txscript/src/lib.rs:574-643): they return the tri-state verdict per triple that the script
engine needs (valid / invalid / pubkey-parse-error / sig-parse-error).

Buffers may be numpy arrays (host path: H2D + kernel + D2H inside the call) or torch CUDA tensors
(device path: enqueued on the current torch stream, no copies, no sync).
"""
import ctypes

import numpy as np

from . import _lib


def _addr_and_keepalive(buf, nbytes, writable=False):
    """Returns (address, is_device, keepalive) for a numpy array / torch tensor / bytes-like."""
    try:
        import torch
    except Exception:  # pragma: no cover
        torch = None
    if torch is not None and isinstance(buf, torch.Tensor):
        if not buf.is_contiguous():
            raise ValueError("tensor must be contiguous")
        if buf.numel() * buf.element_size() < nbytes:
            raise ValueError("tensor too small")
        return buf.data_ptr(), buf.is_cuda, buf
    arr = np.ascontiguousarray(buf) if not isinstance(buf, np.ndarray) else buf
    if not arr.flags["C_CONTIGUOUS"]:
        raise ValueError("array must be C-contiguous")
    if arr.nbytes < nbytes:
        raise ValueError("array too small")
    if writable and not arr.flags["WRITEABLE"]:
        raise ValueError("output array must be writable")
    return arr.ctypes.data, False, arr


class _KgvTxBatch(ctypes.Structure):
    _fields_ = [("txs", ctypes.c_void_p), ("n_txs", ctypes.c_size_t), ("inputs", ctypes.c_void_p), ("n_inputs", ctypes.c_size_t),
                ("outputs", ctypes.c_void_p), ("n_outputs", ctypes.c_size_t), ("entries", ctypes.c_void_p),
                ("bytes", ctypes.c_void_p), ("n_bytes", ctypes.c_size_t)]


SIGHASH_ITEM_DTYPE = np.dtype([("tx", "<u4"), ("input", "<u4"), ("hash_type", "u1"), ("ecdsa", "u1"), ("pad_", "u1", (2,))])
assert SIGHASH_ITEM_DTYPE.itemsize == 12


def _c_batch(b, with_entries=True):
    """ctypes view of a txbatch.TxBatch (host arrays)."""
    cb = _KgvTxBatch(b.txs.ctypes.data, len(b.txs), b.inputs.ctypes.data, len(b.inputs), b.outputs.ctypes.data, len(b.outputs),
                     b.entries.ctypes.data if (with_entries and b.entries is not None) else None, b.arena.ctypes.data, len(b.arena))
    cb._keep = b
    return cb


class GpuContext:
    """One per device; wraps kgv_create/kgv_destroy. Fails loudly without a CUDA device."""

    def __init__(self, device=0):
        self._lib = _lib.load()
        h = ctypes.c_void_p()
        rc = self._lib.kgv_create(int(device), 0, ctypes.byref(h))
        if rc != 0 or not h:
            raise _lib.KgvError(f"kgv_create(device={device}) failed with {rc}: no usable CUDA device (no CPU fallback)")
        self._h = h
        self.device = int(device)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.kgv_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise _lib.KgvError(f"kgv call failed ({rc}): {self._lib.kgv_last_error(self._h).decode()}")

    def use_stream(self, cuda_stream_handle):
        self._check(self._lib.kgv_set_stream(self._h, ctypes.c_void_p(cuda_stream_handle)))

    def use_torch_stream(self):
        import torch
        self.use_stream(torch.cuda.current_stream(self.device).cuda_stream)

    def reset_stream(self):
        """back to the context's private stream"""
        self._check(self._lib.kgv_reset_stream(self._h))

    def synchronize(self):
        self._check(self._lib.kgv_synchronize(self._h))

    @property
    def launch_count(self):
        return int(self._lib.kgv_launch_count(self._h))

    # -- signature batches -------------------------------------------------------------------
    def _verify(self, fn, pk, pk_stride, msg, sig, n, status):
        if status is None:
            status = np.empty(n, dtype=np.uint8)
        a_pk, d0, k0 = _addr_and_keepalive(pk, pk_stride * n)
        a_msg, d1, k1 = _addr_and_keepalive(msg, 32 * n)
        a_sig, d2, k2 = _addr_and_keepalive(sig, 64 * n)
        a_st, d3, k3 = _addr_and_keepalive(status, n, writable=True)
        self._check(fn(self._h, a_pk, a_msg, a_sig, n, a_st))
        return status

    def verify_schnorr_batch(self, pk32, msg32, sig64, n=None, status=None):
        """status[i] in {0 invalid, 1 valid, 2 pubkey parse error} for BIP-340 triples (SoA buffers)."""
        if n is None:
            n = _nbytes(pk32) // 32
        return self._verify(self._lib.kgv_schnorr_verify, pk32, 32, msg32, sig64, n, status)

    def verify_ecdsa_batch(self, pk33, msg32, sig64, n=None, status=None):
        """status[i] in {0,1,2,3} for ECDSA triples with 33-byte compressed keys (SoA buffers)."""
        if n is None:
            n = _nbytes(pk33) // 33
        return self._verify(self._lib.kgv_ecdsa_verify, pk33, 33, msg32, sig64, n, status)

    def status_to_bitmap(self, status, n=None, bitmap=None):
        if n is None:
            n = _nbytes(status)
        if bitmap is None:
            bitmap = np.empty((n + 7) // 8, dtype=np.uint8)
        a_st, _, k0 = _addr_and_keepalive(status, n)
        a_bm, _, k1 = _addr_and_keepalive(bitmap, (n + 7) // 8, writable=True)
        self._check(self._lib.kgv_status_to_bitmap(self._h, a_st, n, a_bm))
        return bitmap

    # -- transaction hashing ----------------------------------------------------------------------
    def tx_ids(self, batch):
        """(n_txs, 32) uint8: Transaction::id() of every tx (consensus/core/src/hashing/tx.rs:30-42)."""
        out = np.zeros((batch.n_txs, 32), dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self._check(self._lib.kgv_tx_ids(self._h, ctypes.byref(cb), out.ctypes.data))
        return out

    def tx_hashes(self, batch):
        """(n_txs, 32) uint8: hashing::tx::hash of every tx (consensus/core/src/hashing/tx.rs:16-20)."""
        out = np.zeros((batch.n_txs, 32), dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self._check(self._lib.kgv_tx_hashes(self._h, ctypes.byref(cb), out.ctypes.data))
        return out

    def merkle_roots(self, hashes32, first):
        """calc_merkle_root (crypto/merkle/src/lib.rs:3-30) of every group of 32-byte hashes: group g = rows [first[g], first[g+1]).
        Returns (n_groups, 32) uint8."""
        h = np.ascontiguousarray(hashes32, dtype=np.uint8).reshape(-1, 32)
        f = np.ascontiguousarray(first, dtype=np.uint32)
        out = np.zeros((len(f) - 1, 32), dtype=np.uint8)
        self._check(self._lib.kgv_merkle_roots(self._h, h.ctypes.data if len(h) else None, f.ctypes.data, len(f) - 1, out.ctypes.data))
        return out

    def block_hash_merkle_roots(self, batch, block_first_tx):
        """calc_hash_merkle_root of every block of the batch (block b = txs [block_first_tx[b], block_first_tx[b+1]))."""
        f = np.ascontiguousarray(block_first_tx, dtype=np.uint32)
        out = np.zeros((len(f) - 1, 32), dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self._check(self._lib.kgv_block_hash_merkle_roots(self._h, ctypes.byref(cb), f.ctypes.data, len(f) - 1, out.ctypes.data))
        return out

    def block_set_checks(self, batch, block_first_tx):
        """duplicate-tx / double-spend / chained-tx checks of validate_body_in_isolation for every block of the batch.
        Returns a structured array (status, index), see KGV_BLOCK_* in include/kgv.h."""
        f = np.ascontiguousarray(block_first_tx, dtype=np.uint32)
        out = np.zeros(len(f) - 1, dtype=np.dtype([("status", "<u4"), ("index", "<u4")]))
        cb = _c_batch(batch, with_entries=False)
        self._check(self._lib.kgv_block_set_checks(self._h, ctypes.byref(cb), f.ctypes.data, len(f) - 1, out.ctypes.data))
        return out

    def sighash(self, batch, items):
        """items: array of SIGHASH_ITEM_DTYPE or list of (tx, abs_input, hash_type, ecdsa). Returns (n, 32) uint8."""
        if not isinstance(items, np.ndarray):
            arr = np.zeros(len(items), dtype=SIGHASH_ITEM_DTYPE)
            for i, (t, a, h, e) in enumerate(items):
                arr[i] = (t, a, h, 1 if e else 0, (0, 0))
            items = arr
        out = np.zeros((len(items), 32), dtype=np.uint8)
        cb = _c_batch(batch)
        self._check(self._lib.kgv_sighash(self._h, ctypes.byref(cb), items.ctypes.data, len(items), out.ctypes.data))
        return out

    def debug_selftest(self, op, a_vals, b_vals):
        """Runs arithmetic primitive `op` (include/kgv.h) on the device for lists of 256-bit ints; returns 512-bit ints."""
        n = len(a_vals)
        inp = np.zeros((n, 16), dtype=np.uint32)
        for i, (a, b) in enumerate(zip(a_vals, b_vals)):
            for k in range(8):
                inp[i, k] = (a >> (32 * k)) & 0xFFFFFFFF
                inp[i, 8 + k] = (b >> (32 * k)) & 0xFFFFFFFF
        out = np.zeros((n, 16), dtype=np.uint32)
        self._check(self._lib.kgv_debug_selftest(self._h, int(op), inp.ctypes.data, out.ctypes.data, n))
        return [sum(int(out[i, k]) << (32 * k) for k in range(16)) for i in range(n)]

    def debug_schnorr_trace(self, pk32, msg32, sig64):
        """(status, trace[32][16] uint32) of one triple verified on the device (audit hook)."""
        tr = np.zeros((_lib.TRACE_STAGES, 16), dtype=np.uint32)
        st = np.zeros(1, dtype=np.uint8)
        bufs = [np.frombuffer(bytes(b), dtype=np.uint8).copy() for b in (pk32, msg32, sig64)]
        self._check(self._lib.kgv_debug_schnorr_trace(self._h, bufs[0].ctypes.data, bufs[1].ctypes.data, bufs[2].ctypes.data,
                                                      tr.ctypes.data, st.ctypes.data))
        return int(st[0]), tr

    def debug_key_form(self, ecdsa=False):
        """Key form of the last non-indexed verify launch of one kind (audit hook, synchronises): dict with n_items, threads,
        distinct_keys and form, one of "no-cache", "inline", "plain", "comb" (KGV_KEY_FORM_* in include/kgv.h)."""
        info = _lib.KeyFormInfo()
        self._check(self._lib.kgv_debug_key_form(self._h, 1 if ecdsa else 0, ctypes.byref(info)))
        return {"n_items": int(info.n_items), "threads": int(info.threads), "distinct_keys": int(info.distinct_keys),
                "form": _lib.KEY_FORMS[info.form]}

    def gtable_entry(self, which, v):
        out = (ctypes.c_uint8 * 64)()
        self._check(self._lib.kgv_gtable_entry(self._h, which, v, ctypes.addressof(out)))
        b = bytes(out)
        return int.from_bytes(b[:32], "big"), int.from_bytes(b[32:], "big")


def _nbytes(buf):
    if hasattr(buf, "nbytes"):
        return int(buf.nbytes)
    if hasattr(buf, "numel"):
        return int(buf.numel() * buf.element_size())
    return len(buf)
