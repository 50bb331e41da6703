"""DAG replay on the GPU: the caller side of the hot path (SURVEY.md §8a-18: calculate_utxo_state /
verify_expected_utxo_state, consensus/src/pipeline/virtual_processor/utxo_validation.rs:110-228).

Two schedules with identical results:

  blockwise   for every (merged) block in order: validate_transactions_in_parallel(Full) against the UTXO
              table, then UtxoDiff::add_transaction for the accepted ones.  This is the reference's order; a
              10-BPS block carries <= ~300 signatures, far too few to fill an H100.

  windowed    ONE library call per window of blocks (kgv_replay_window, include/kgv.h): every script of the window
              is checked in one large batch (signatures are context free given the spent output, SURVEY §0-6; outputs
              created inside the window are resolved on the device), then a single persistent kernel walks the
              blocks in order: populate, UTXO-context rules, accept = context ok AND scripts ok, erase / insert.
              Nothing of the schedule lives in Python any more: this module only flattens the blocks into the
              batch layout and names the per-block flags.
"""
import ctypes

import numpy as np

from .txbatch import ENTRY_DTYPE, TxBatch, build_batch
from .validator import FLAGS_FULL, RESULT_DTYPE, TX_OK, TX_SKIPPED_COINBASE, GpuUtxoSet, TransactionValidator
from .verifier import _c_batch

REPLAY_BLOCK_DTYPE = np.dtype([("first_tx", "<u4"), ("n_txs", "<u4"), ("pov_daa_score", "<u8"), ("flags", "<u4"), ("pad_", "<u4")])
assert REPLAY_BLOCK_DTYPE.itemsize == 24
REPLAY_ACCEPT_COINBASE, REPLAY_SKIP_SCRIPTS, REPLAY_VERIFY_ONLY = 1, 2, 4

# kgv_replay_verify_chain (include/kgv.h)
CHAIN_HEADER_DTYPE = np.dtype([("utxo_commitment", "u1", 32), ("accepted_id_merkle_root", "u1", 32), ("selected_parent_accepted_id_merkle_root", "u1", 32),
                               ("blue_score", "<u8"), ("expected_subsidy", "<u8")])
assert CHAIN_HEADER_DTYPE.itemsize == 112
CHAIN_RESULT_DTYPE = np.dtype([("status", "<u4"), ("n_invalid_txs", "<u4"), ("n_txs", "<u4"), ("pad_", "<u4"), ("utxo_commitment", "u1", 32),
                               ("accepted_id_merkle_root", "u1", 32), ("coinbase_hash", "u1", 32)])
assert CHAIN_RESULT_DTYPE.itemsize == 112
CHAIN_STATUS = {"Ok": 0, "BadUTXOCommitment": 1, "BadAcceptedIDMerkleRoot": 2, "BadCoinbaseTransaction": 3, "RewardOverflow": 4, "CoinbasePayloadUnparsable": 5}
MERGED_RED, MERGED_NON_DAA = 1, 2


class ReplayStats(ctypes.Structure):
    _fields_ = [("n_accepted", ctypes.c_uint64), ("n_sig_checks", ctypes.c_uint64), ("n_host_vm", ctypes.c_uint64), ("pre_check_ms", ctypes.c_float),
                ("in_order_ms", ctypes.c_float)]


def replay_blocks_array(ranges):
    """ranges: iterable of (first_tx, n_txs, pov_daa_score, flags) -> REPLAY_BLOCK_DTYPE array"""
    ranges = list(ranges)
    a = np.zeros(len(ranges), dtype=REPLAY_BLOCK_DTYPE)
    for i, (f, n, pov, fl) in enumerate(ranges):
        a[i] = (f, n, pov, fl, 0)
    return a


class ReplayDiffs:
    """What kgv_replay_diffs returns: per group g (ranges[g] = first_remove, n_remove, first_add, n_add) its removals (outpoint keys and the
    entries they had) and additions, in window order; every entry's script_off points into `bytes`."""

    def __init__(self, ranges, rem_keys36, rem_entries, add_keys36, add_entries, arena):
        self.ranges, self.rem_keys36, self.rem_entries, self.add_keys36, self.add_entries, self.bytes = ranges, rem_keys36, rem_entries, add_keys36, add_entries, arena

    def __len__(self):
        return len(self.ranges)

    def group(self, g):
        """(rem_keys36, rem_entries, add_keys36, add_entries) of group g (views into the whole arrays)"""
        fr, nr, fa, na = (int(x) for x in self.ranges[g])
        return self.rem_keys36[fr:fr + nr], self.rem_entries[fr:fr + nr], self.add_keys36[fa:fa + na], self.add_entries[fa:fa + na]

    def utxo_diff(self, g):
        """group g as a utxo_diff.UtxoDiff (outpoint (txid, index) -> entry dict)"""
        from .utxo_diff import UtxoDiff

        def coll(keys, ents):
            out = {}
            for k, e in zip(keys, ents):
                off, n = int(e["script_off"]), int(e["script_len"])
                out[(k[:32].tobytes(), int.from_bytes(k[32:].tobytes(), "little"))] = {
                    "amount": int(e["amount"]), "spk_version": int(e["spk_version"]), "script": self.bytes[off:off + n].tobytes(),
                    "block_daa_score": int(e["block_daa_score"]), "is_coinbase": bool(e["is_coinbase"])}
            return out
        rk, re, ak, ae = self.group(g)
        return UtxoDiff(add=coll(ak, ae), remove=coll(rk, re))

    def apply(self, utxo_set, g, reverse=False):
        """write group g's diff into a GpuUtxoSet or view (kgv_utxo_apply_diff); reverse=True undoes it (UtxoDiff::as_reversed, processor.rs:395-397).
        Returns (rem_status, add_status): 1 = was present / inserted."""
        rk, re, ak, ae = self.group(g)
        if reverse:
            rk, (ak, ae) = ak, (rk, re)
        ae = ae.copy()
        lo = int(ae["script_off"].min()) if len(ae) else 0
        hi = int((ae["script_off"].astype(np.int64) + ae["script_len"]).max()) if len(ae) else 0
        ae["script_off"] -= lo  # the group's scripts are one contiguous range of the arena: hand over only that
        return utxo_set.apply_diff(rem_keys36=rk if len(rk) else None, add_keys36=ak if len(ak) else None, add_entries=ae if len(ae) else None,
                                   add_bytes=np.concatenate([self.bytes[lo:hi], np.zeros(8, np.uint8)]))


class DagReplayer:
    """Replays a linearised schedule of blocks.  Every block is given as (txs, pov_daa_score[, flags]); txs[0] is the
    block's coinbase (skipped by position, utxo_validation.rs:273).  flags default to REPLAY_ACCEPT_COINBASE: the
    generated schedules are chains (one merged block = the selected parent per chain block, its coinbase accepted,
    utxo_validation.rs:116-121) that are nevertheless fully script-checked.  For a real DAG the caller marks only the
    selected parent of each mergeset with ACCEPT_COINBASE | SKIP_SCRIPTS and gives all merged blocks the chain block's
    pov_daa_score (tests/test_gpu_replay.py replays the reference's simpa fixtures that way)."""

    def __init__(self, ctx, params, capacity_slots=1 << 20, max_load=None):
        """max_load: growth policy of the UTXO table in permille (GpuUtxoSet.set_max_load); None keeps the table at capacity_slots"""
        self.ctx = ctx
        self.tv = TransactionValidator(ctx, params)
        self.us = GpuUtxoSet(ctx, capacity_slots)
        if max_load is not None:
            self.us.set_max_load(max_load)
        self.last_stats = None

    def close(self):
        self.us.close()

    # ---------------------------------------------------------------------------------------- blockwise
    def replay_blockwise(self, blocks, multiset=None):
        """Returns the list of per-block RESULT arrays.
        multiset: optional MuHash that follows the UTXO set the way UtxoProcessingContext.multiset_hash does
        (utxo_validation.rs:120,144): the accepted coinbase and every accepted transaction of each block are combined into it."""
        from .muhash import MuHash
        out = []
        for blk in blocks:
            txs, pov = blk[0], blk[1]
            flags = blk[2] if len(blk) > 2 else REPLAY_ACCEPT_COINBASE
            b = txs if isinstance(txs, TxBatch) else build_batch(txs)
            vflags = 1 if (flags & REPLAY_SKIP_SCRIPTS) else FLAGS_FULL
            res = self.tv.validate_transactions_in_parallel(self.us, b, pov, vflags)  # non-standard scripts are decided inside the call
            res["status"][0] = TX_SKIPPED_COINBASE  # position 0 is the coinbase
            acc = (res["status"] == TX_OK).astype(np.uint8)
            acc[0] = 1 if (flags & REPLAY_ACCEPT_COINBASE) else 0
            if flags & REPLAY_VERIFY_ONLY:
                acc[:] = 0
            if multiset is not None and acc.any():  # before the spent entries are erased
                multiset.combine(MuHash.from_transactions(self.ctx, b, acc, pov, utxo_set=self.us))
            if acc.any():
                self.us.add_transactions(b, acc, pov)
            out.append(res)
        return out

    # ---------------------------------------------------------------------------------------- windowed
    def replay_window(self, batch, blocks_arr, want_accept=False):
        """One kgv_replay_window call on a flattened batch; returns RESULT_DTYPE[n_txs] (and the accept mask)."""
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        acc = np.zeros(batch.n_txs, dtype=np.uint8)
        st = ReplayStats()
        cb = _c_batch(batch, with_entries=False)
        blocks_arr = np.ascontiguousarray(blocks_arr, dtype=REPLAY_BLOCK_DTYPE)
        self.ctx._check(self.ctx._lib.kgv_replay_window(self.ctx._h, self.us._h, ctypes.byref(cb), blocks_arr.ctypes.data, len(blocks_arr),
                                                        ctypes.byref(self.tv.params), res.ctypes.data, acc.ctypes.data, ctypes.byref(st)))
        self.last_stats = {"n_accepted": int(st.n_accepted), "n_sig_checks": int(st.n_sig_checks), "n_host_vm": int(st.n_host_vm), "pre_check_ms": float(st.pre_check_ms),
                           "in_order_ms": float(st.in_order_ms)}
        return (res, acc) if want_accept else res

    def prefetch(self, batch):
        """kgv_batch_prefetch: start uploading the NEXT window's (host) batch while the current window computes; the replay_window call that gets
        this very batch object then skips its upload"""
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self.ctx._lib.kgv_batch_prefetch(self.ctx._h, ctypes.byref(cb)))

    def replay_muhash(self, group_first_block):
        """kgv_replay_muhash for the window just replayed: (n_groups, 768) uint8 (numerator || denominator) of what each group of blocks accepted"""
        gf = np.ascontiguousarray(group_first_block, dtype=np.uint32)
        out = np.zeros((len(gf) - 1, 768), dtype=np.uint8)
        if len(gf) > 1:
            self.ctx._check(self.ctx._lib.kgv_replay_muhash(self.ctx._h, gf.ctypes.data, len(gf) - 1, out.ctypes.data))
        return out

    def replay_diffs(self, group_first_block):
        """kgv_replay_diffs for the window just replayed: the UtxoDiff of every group of blocks (ctx.mergeset_diff, utxo_validation.rs:119,148)"""
        gf = np.ascontiguousarray(group_first_block, dtype=np.uint32)
        n_groups = len(gf) - 1
        lib, h = self.ctx._lib, self.ctx._h
        ranges = np.zeros((max(n_groups, 1), 4), dtype=np.uint64)
        nr, na, nb = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        self.ctx._check(lib.kgv_replay_diffs(h, gf.ctypes.data, n_groups, ranges.ctypes.data, None, None, None, None, None, 0, 0, 0,
                                             ctypes.byref(nr), ctypes.byref(na), ctypes.byref(nb)))
        rk = np.zeros((max(nr.value, 1), 36), dtype=np.uint8)
        re = np.zeros(max(nr.value, 1), dtype=ENTRY_DTYPE)
        ak = np.zeros((max(na.value, 1), 36), dtype=np.uint8)
        ae = np.zeros(max(na.value, 1), dtype=ENTRY_DTYPE)
        by = np.zeros(max(nb.value, 8), dtype=np.uint8)
        self.ctx._check(lib.kgv_replay_diffs(h, gf.ctypes.data, n_groups, ranges.ctypes.data, rk.ctypes.data, re.ctypes.data, ak.ctypes.data, ae.ctypes.data,
                                             by.ctypes.data, nr.value, na.value, nb.value, ctypes.byref(nr), ctypes.byref(na), ctypes.byref(nb)))
        return ReplayDiffs(ranges[:n_groups], rk[:nr.value], re[:nr.value], ak[:na.value], ae[:na.value], by[:nb.value])

    def verify_chain(self, group_first, headers, merged_flags, init768, rules=None, body_rules=None):
        """kgv_replay_verify_chain for the window just replayed: verify_expected_utxo_state of every chain block (utxo_validation.rs:182-228).
        group_first: n_groups + 1 block offsets; group g is the chain block's selected parent (ACCEPT_COINBASE), the rest of its mergeset in
        consensus order, then its own body (VERIFY_ONLY).  headers: CHAIN_HEADER_DTYPE per group; merged_flags: MERGED_* per window block;
        init768: the multiset of the window's first selected parent (a MuHash, or 768 bytes numerator || denominator).
        Returns (CHAIN_RESULT_DTYPE[n_groups], block_fees uint64[n_blocks], (n_groups, 768) uint8 running multisets)."""
        from .validator import BodyRules, TxRules
        gf = np.ascontiguousarray(group_first, dtype=np.uint32)
        h = np.ascontiguousarray(headers, dtype=CHAIN_HEADER_DTYPE)
        mf = np.ascontiguousarray(merged_flags, dtype=np.uint8)
        if hasattr(init768, "numerator"):  # a MuHash
            init768 = init768.numerator + init768.denominator
        init = np.frombuffer(bytes(init768), dtype=np.uint8).copy() if isinstance(init768, (bytes, bytearray)) else np.ascontiguousarray(init768, dtype=np.uint8)
        n_groups = len(gf) - 1
        # the call reads one merged-flags byte and writes one fee per window block (group_first[-1] of them), and reads one header per group
        if n_groups < 1 or len(h) != n_groups or len(mf) != int(gf[-1]) or init.size != 768:
            raise ValueError("one header per group, one merged-flags byte per window block and a 768-byte init multiset")
        rules, body_rules = rules or TxRules(), body_rules or BodyRules()
        res = np.zeros(max(n_groups, 1), dtype=CHAIN_RESULT_DTYPE)
        fees = np.zeros(max(len(mf), 1), dtype=np.uint64)
        ms = np.zeros((max(n_groups, 1), 768), dtype=np.uint8)
        self.ctx._check(self.ctx._lib.kgv_replay_verify_chain(self.ctx._h, gf.ctypes.data, n_groups, h.ctypes.data, mf.ctypes.data, init.ctypes.data,
                                                              ctypes.byref(rules), ctypes.byref(body_rules), res.ctypes.data, fees.ctypes.data, ms.ctypes.data))
        return res[:n_groups], fees[:len(mf)], ms[:n_groups]

    def replay_windowed(self, blocks):
        """blocks: list of (txs, pov[, flags]) forming ONE window. Returns per-block RESULT arrays (same values as blockwise)."""
        blocks = list(blocks)
        all_txs, ranges = [], []
        for blk in blocks:
            txs, pov = blk[0], blk[1]
            flags = blk[2] if len(blk) > 2 else REPLAY_ACCEPT_COINBASE
            ranges.append((len(all_txs), len(txs), pov, flags))
            all_txs.extend(txs)
        b = build_batch(all_txs)
        res = self.replay_window(b, replay_blocks_array(ranges))
        return [res[f:f + n] for f, n, _, _ in ranges]
