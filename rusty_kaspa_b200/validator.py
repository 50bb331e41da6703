"""Host-side Python mirror of the validation surface of the reference, on top of the C ABI.

    TransactionValidator.validate_populated_transactions  <->  validate_populated_transaction_and_get_fee
        (consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs:34-61)
    GpuUtxoSet (get / apply_diff / count / digest)          <->  UtxoView::get, DbUtxoSetStore::write_diff_batch
        (consensus/core/src/utxo/utxo_view.rs:5-7, consensus/src/model/stores/utxo_set.rs:107-112,143-152)
    TransactionValidator.validate_transactions_in_parallel  <->  VirtualStateProcessor::validate_transactions_in_parallel
        (consensus/src/pipeline/virtual_processor/utxo_validation.rs:262-278)
    TransactionValidator.validate_mempool_transactions_in_utxo_context  <->  validate_mempool_transaction_in_utxo_context
        (utxo_validation.rs:341-397), for a batch
    TransactionValidator.validate_txs_in_isolation           <->  validate_tx_in_isolation + validate_tx_in_header_context_with_args
        (tx_validation_in_isolation.rs:16-26, tx_validation_in_header_context.rs) and calc_non_contextual_masses (mass/mod.rs:248-269)
    TransactionValidator.validate_mempool_transactions_in_parallel_full  <->  validate_mempool_transactions_in_parallel
        (processor.rs:853-878): isolation -> finality -> UTXO context, per transaction
    TransactionValidator.check_transaction_standard_in_isolation / check_transaction_standard_in_context / is_transaction_output_dust
        <->  Mempool::check_transaction_standard_in_isolation / _in_context / is_transaction_output_dust
        (mining/src/mempool/check_transaction_standard.rs:41-211), for a batch
    TransactionValidator.validate_mempool_transactions_with_policy  <->  the mempool's admission order with its standardness policy
        (mining/src/mempool/validate_and_insert_transaction.rs:20-33, 142-159)
    GpuUtxoSet.add_transactions                              <->  UtxoDiff::add_transaction (utxo_diff.rs:233-247)
    BlockBodyProcessor.validate_body_in_isolation / validate_body_in_context / validate_bodies  <->  BlockBodyProcessor
        (consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:13-131, body_validation_in_context.rs:20-80), a window per call
"""
import ctypes

import numpy as np

from . import _lib
from .txbatch import ENTRY_DTYPE, TxBatch
from .verifier import _c_batch

RESULT_DTYPE = np.dtype([("fee", "<u8"), ("fail_input", "<u4"), ("status", "u1"), ("script_err", "u1"), ("pad_", "u1", (2,))])
assert RESULT_DTYPE.itemsize == 16
MEMPOOL_ARGS_DTYPE = np.dtype([("feerate_threshold", "<f8"), ("non_contextual_mass", "<u8")])  # kgv_mempool_tx_args
assert MEMPOOL_ARGS_DTYPE.itemsize == 16
TX_MASSES_DTYPE = np.dtype([("compute_mass", "<u8"), ("transient_mass", "<u8")])  # kgv_tx_masses
assert TX_MASSES_DTYPE.itemsize == 16
ISOLATION_SKIP_FINALITY = 1
# KGV_TX_* verdicts of the isolation and finality rules (include/kgv.h), by the reference's TxRuleError names
ISOLATION_STATUS = {14: "NoTxInputs", 15: "TooManyInputs", 16: "TooBigSignatureScript", 17: "TooManyOutputs", 18: "TooBigScriptPublicKey",
                    19: "CoinbaseHasInputs", 20: "CoinbaseNonZeroMassCommitment", 21: "CoinbaseTooManyOutputs",
                    22: "CoinbaseScriptPublicKeyTooLong", 23: "TxOutZero", 24: "TxOutTooHigh", 25: "OutputsValueOverflow",
                    26: "TotalTxOutTooHigh", 27: "TxDuplicateInputs", 28: "TxHasGas", 29: "SubnetworksDisabled", 30: "UnknownTxVersion",
                    31: "NotFinalized"}
# KGV_TX_* verdicts of the standardness policy (include/kgv.h), by the reference's NonStandardError names
STANDARD_STATUS = {32: "RejectVersion", 33: "RejectComputeMass", 34: "RejectTransientMass", 35: "RejectSignatureScriptSize",
                   36: "RejectScriptPublicKeyVersion", 37: "RejectOutputScriptClass", 38: "RejectDust", 39: "RejectStorageMass",
                   40: "RejectInputScriptClass", 41: "RejectSignatureCount", 42: "RejectInsufficientFee"}

# kgv_block_header_ctx / kgv_body_result / kgv_block_masses
BLOCK_HEADER_CTX_DTYPE = np.dtype([("hash_merkle_root", "u1", (32,)), ("daa_score", "<u8"), ("blue_score", "<u8"), ("past_median_time", "<u8"),
                                   ("expected_subsidy", "<u8")])
BODY_RESULT_DTYPE = np.dtype([("status", "<u4"), ("index", "<u4"), ("tx_status", "<u4"), ("fail_input", "<u4"), ("a", "<u8"), ("b", "<u8")])
BLOCK_MASSES_DTYPE = np.dtype([("compute_mass", "<u8"), ("transient_mass", "<u8"), ("storage_mass", "<u8")])
assert (BLOCK_HEADER_CTX_DTYPE.itemsize, BODY_RESULT_DTYPE.itemsize, BLOCK_MASSES_DTYPE.itemsize) == (64, 32, 24)
BODY_ISOLATION_ONLY = 1
# KGV_BODY_* verdicts (include/kgv.h), by the reference's RuleError names
BODY_STATUS = {0: "Ok", 1: "NoTransactions", 2: "BadMerkleRoot", 3: "FirstTxNotCoinbase", 4: "MultipleCoinbases", 5: "TxInIsolationValidationFailed",
               6: "ExceedsComputeMassLimit", 7: "ExceedsTransientMassLimit", 8: "ExceedsStorageMassLimit", 9: "DuplicateTransactions",
               10: "DoubleSpendInSameBlock", 11: "ChainedTransaction", 12: "BadCoinbasePayload", 13: "BadCoinbasePayloadBlueScore", 14: "WrongSubsidy",
               15: "TxInContextFailed"}

FLAGS_FULL, FLAGS_SKIP_SCRIPT_CHECKS, FLAGS_SKIP_MASS_CHECK, FLAGS_SCRIPTS_ONLY = 0, 1, 2, 3
MAX_SOMPI = 29_000_000_000 * 100_000_000
TX_OK, TX_NEEDS_HOST_VM, TX_SKIPPED_COINBASE, TX_FEERATE_TOO_LOW = 0, 11, 12, 13
ERR_NOMEM = -3


class Params(ctypes.Structure):
    """kgv_params: the consensus parameters the path reads (consensus/core/src/config/params.rs)."""
    _fields_ = [("coinbase_maturity", ctypes.c_uint64), ("storage_mass_parameter", ctypes.c_uint64), ("max_sompi", ctypes.c_uint64)]

    def __init__(self, coinbase_maturity=100, storage_mass_parameter=10**12, max_sompi=MAX_SOMPI):
        super().__init__(coinbase_maturity, storage_mass_parameter, max_sompi)


class TxRules(ctypes.Structure):
    """kgv_tx_rules: the parameters of the isolation rules and the non-contextual masses.  The defaults are mainnet's
    (MAINNET_PARAMS, consensus/core/src/config/params.rs; ghostdag_k of the 10 BPS blockrate)."""
    _fields_ = [(n, ctypes.c_uint64) for n in ("max_tx_inputs", "max_tx_outputs", "max_signature_script_len", "max_script_public_key_len",
                                               "mass_per_tx_byte", "mass_per_script_pub_key_byte", "mass_per_sig_op", "ghostdag_k",
                                               "coinbase_payload_script_public_key_max_len")]
    MAINNET = dict(max_tx_inputs=1000, max_tx_outputs=1000, max_signature_script_len=10_000, max_script_public_key_len=10_000, mass_per_tx_byte=1,
                   mass_per_script_pub_key_byte=10, mass_per_sig_op=1000, ghostdag_k=124, coinbase_payload_script_public_key_max_len=150)

    def __init__(self, **overrides):
        unknown = set(overrides) - set(self.MAINNET)
        if unknown:
            raise TypeError("unknown rule parameters: %s" % sorted(unknown))
        super().__init__(**{**self.MAINNET, **overrides})


assert ctypes.sizeof(TxRules) == 72


class MempoolPolicy(ctypes.Structure):
    """kgv_mempool_policy: the mempool Config fields the standardness policy reads (mining/src/mempool/config.rs); the defaults are the
    reference's (DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE, and TX_VERSION for both versions)."""
    _fields_ = [("minimum_relay_transaction_fee", ctypes.c_uint64), ("minimum_standard_transaction_version", ctypes.c_uint16),
                ("maximum_standard_transaction_version", ctypes.c_uint16), ("pad_", ctypes.c_uint8 * 4)]

    def __init__(self, minimum_relay_transaction_fee=1000, minimum_standard_transaction_version=0, maximum_standard_transaction_version=0):
        super().__init__(minimum_relay_transaction_fee, minimum_standard_transaction_version, maximum_standard_transaction_version)


assert ctypes.sizeof(MempoolPolicy) == 16


class SigRequest(ctypes.Structure):
    """kgv_sig_request: one signature check the host script engine asks a verdict for."""
    _fields_ = [("tx", ctypes.c_uint32), ("input", ctypes.c_uint32), ("hash_type", ctypes.c_uint8), ("ecdsa", ctypes.c_uint8), ("key_len", ctypes.c_uint8),
                ("pad_", ctypes.c_uint8), ("key", ctypes.c_uint8 * 33), ("sig", ctypes.c_uint8 * 64), ("pad2_", ctypes.c_uint8 * 3)]


assert ctypes.sizeof(SigRequest) == 112
VERDICT_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(SigRequest))

SCRIPT_ERR_NAMES = {0: "Ok", 1: "EvalFalse", 2: "NullFail", 3: "InvalidSignature", 4: "SigLength", 5: "PubKeyFormat", 6: "InvalidSigHashType",
                    7: "ExceededSigOpLimit", 8: "SignatureScriptNotPushOnly", 9: "CleanStack", 10: "EmptyStack", 11: "ElementTooBig",
                    12: "TooManyOperations", 13: "StackSizeExceeded", 14: "OpcodeDisabled", 15: "OpcodeReserved", 16: "InvalidOpcode",
                    17: "MalformedPush", 18: "MalformedPushSize", 19: "NotMinimalData", 20: "ErrUnbalancedConditional",
                    21: "InvalidState(condition stack empty)", 22: "InvalidState(expected boolean)", 23: "InvalidState(pick at an invalid location)",
                    24: "InvalidState(roll at an invalid location)", 25: "VerifyError", 26: "EarlyReturn", 27: "InvalidStackOperation", 28: "NumberTooBig",
                    29: "InvalidPubKeyCount", 30: "InvalidSignatureCount", 31: "UnsatisfiedLockTime", 32: "ScriptSize", 33: "NoScripts",
                    34: "InvalidInputIndex", 35: "InvalidOutputIndex", 36: "Serialization", 254: "NeedsSigVerdicts", 255: "NonStandard"}


def script_execute(batch, tx, input_index, verdict=None):
    """TxScriptEngine::from_transaction_input(..).execute() on the HOST engine of libkgv (no GPU involved).
    verdict(request: SigRequest) -> KGV_SIG_* or -1.  Returns the KGV_SCRIPT_* code."""
    lib = _lib.load()
    cb = _c_batch(batch, with_entries=True)
    fn = VERDICT_FN((lambda user, rq: int(verdict(rq.contents))) if verdict else (lambda user, rq: -1))
    err = ctypes.c_uint8(0)
    rc = lib.kgv_script_execute(ctypes.byref(cb), int(tx), int(input_index), ctypes.cast(fn, ctypes.c_void_p), None, ctypes.addressof(err))
    if rc != 0:
        raise _lib.KgvError(f"kgv_script_execute failed ({rc})")
    return int(err.value)


class UtxoTableStats(ctypes.Structure):
    """kgv_utxo_table_stats"""
    _fields_ = [(n, ctypes.c_uint64) for n in ("capacity_slots", "live", "tombstones", "empty", "overflow_used", "overflow_cap", "overflow_live",
                                               "insert_failures", "rehashes", "max_displacement", "sum_displacement", "longest_run")]


assert ctypes.sizeof(UtxoTableStats) == 96


class GpuUtxoSet:
    """GPU-resident UTXO set (kgv_utxo_table)."""

    def __init__(self, ctx, capacity_slots=1 << 20):
        self.ctx = ctx
        self._lib = ctx._lib
        h = ctypes.c_void_p()
        ctx._check(self._lib.kgv_utxo_create(ctx._h, int(capacity_slots), ctypes.byref(h)))
        self._h = h

    def close(self):
        if self._h and getattr(self, "_owner", True):
            self._lib.kgv_utxo_destroy(self.ctx._h, self._h)
        self._h = None

    def on(self, ctx):
        """This same table with its calls issued on `ctx`, another context of its device (include/kgv.h, Threading).  The returned object
        does not own the table: close() on it only drops the handle."""
        v = GpuUtxoSet.__new__(GpuUtxoSet)
        v.__dict__.update(self.__dict__)
        v.ctx, v._owner = ctx, False
        return v

    # ---- composed views (utxo_view.rs:22-35): a diff layer over this set
    def compose(self, capacity_slots=1 << 16):
        """UtxoViewComposition::compose: a GpuUtxoSet that behaves as self ∘ (an initially empty diff); writes through it never touch self"""
        v = GpuUtxoSet.__new__(GpuUtxoSet)
        v.ctx, v._lib = self.ctx, self._lib
        h = ctypes.c_void_p()
        self.ctx._check(self._lib.kgv_utxo_view_create(self.ctx._h, self._h, int(capacity_slots), ctypes.byref(h)))
        v._h, v.base = h, self
        return v

    def commit(self):
        """fold this diff layer into the set below it (write_diff_batch) and empty it"""
        self.ctx._check(self._lib.kgv_utxo_view_commit(self.ctx._h, self._h))

    def discard(self):
        self.ctx._check(self._lib.kgv_utxo_view_discard(self.ctx._h, self._h))

    def get(self, keys36, script_stride=128):
        """keys36: (n, 36) uint8. Returns (found (n,), entries (n,) ENTRY_DTYPE, scripts (n, stride))."""
        keys36 = np.ascontiguousarray(keys36, dtype=np.uint8).reshape(-1, 36)
        n = len(keys36)
        ent = np.zeros(n, dtype=ENTRY_DTYPE)
        scr = np.zeros((n, script_stride), dtype=np.uint8)
        found = np.zeros(n, dtype=np.uint8)
        if n:
            self.ctx._check(self._lib.kgv_utxo_lookup(self.ctx._h, self._h, keys36.ctypes.data, n, ent.ctypes.data, scr.ctypes.data, script_stride, found.ctypes.data))
        return found, ent, scr

    def apply_diff(self, rem_keys36=None, add_keys36=None, add_entries=None, add_bytes=None):
        """write_diff_batch: delete `rem_keys36`, then put (add_keys36, add_entries[script_off/len into add_bytes])."""
        rk = np.zeros((0, 36), np.uint8) if rem_keys36 is None else np.ascontiguousarray(rem_keys36, dtype=np.uint8).reshape(-1, 36)
        ak = np.zeros((0, 36), np.uint8) if add_keys36 is None else np.ascontiguousarray(add_keys36, dtype=np.uint8).reshape(-1, 36)
        ae = np.zeros(0, ENTRY_DTYPE) if add_entries is None else np.ascontiguousarray(add_entries)
        ab = np.zeros(8, np.uint8) if add_bytes is None else np.ascontiguousarray(add_bytes, dtype=np.uint8)
        rs, as_ = np.zeros(max(len(rk), 1), np.uint8), np.zeros(max(len(ak), 1), np.uint8)
        self.ctx._check(self._lib.kgv_utxo_apply_diff(self.ctx._h, self._h, rk.ctypes.data if len(rk) else None, len(rk), rs.ctypes.data,
                                                      ak.ctypes.data if len(ak) else None, ae.ctypes.data if len(ak) else None, ab.ctypes.data, len(ab), len(ak),
                                                      as_.ctypes.data))
        return rs[:len(rk)], as_[:len(ak)]

    def add_transactions(self, batch, accept, pov_daa_score):
        """UtxoDiff::add_transaction for every tx with accept[i] != 0, applied to the table."""
        acc = np.ascontiguousarray(accept, dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_utxo_apply_accepted(self.ctx._h, self._h, ctypes.byref(cb), acc.ctypes.data, int(pov_daa_score)))

    def count(self):
        c = ctypes.c_uint64()
        self.ctx._check(self._lib.kgv_utxo_count(self.ctx._h, self._h, ctypes.byref(c)))
        return int(c.value)

    def digest(self):
        out = (ctypes.c_uint8 * 32)()
        self.ctx._check(self._lib.kgv_utxo_digest(self.ctx._h, self._h, ctypes.addressof(out)))
        return bytes(out)

    # ---- maintenance: churn leaves tombstones and dead arena bytes behind; a rehash drops them
    def stats(self):
        """kgv_utxo_stats: counters and one pass over the slots (of this layer alone for a view), as a dict"""
        s = UtxoTableStats()
        self.ctx._check(self._lib.kgv_utxo_stats(self.ctx._h, self._h, ctypes.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in UtxoTableStats._fields_}

    def rehash(self, capacity=0):
        """kgv_utxo_rehash: rebuild into `capacity` slots (0: the current size; rounded up to a power of two)"""
        self.ctx._check(self._lib.kgv_utxo_rehash(self.ctx._h, self._h, int(capacity)))

    def set_max_load(self, permille):
        """kgv_utxo_set_max_load: 0 = off (the default), 1..900 = grow / rehash before a write would pass that load"""
        self.ctx._check(self._lib.kgv_utxo_set_max_load(self.ctx._h, self._h, int(permille)))

    def export(self):
        """DbUtxoSetStore::iterator (utxo_set.rs:114-129): every live entry. Returns (keys36 (n, 36), entries (n,) ENTRY_DTYPE, arena bytes)."""
        n, nb = ctypes.c_size_t(), ctypes.c_size_t()
        self.ctx._check(self._lib.kgv_utxo_export(self.ctx._h, self._h, None, None, None, 0, 0, ctypes.byref(n), ctypes.byref(nb)))
        keys = np.zeros((max(n.value, 1), 36), dtype=np.uint8)
        ent = np.zeros(max(n.value, 1), dtype=ENTRY_DTYPE)
        arena = np.zeros(max(nb.value, 8), dtype=np.uint8)
        self.ctx._check(self._lib.kgv_utxo_export(self.ctx._h, self._h, keys.ctypes.data, ent.ctypes.data, arena.ctypes.data, n.value, nb.value, ctypes.byref(n), ctypes.byref(nb)))
        return keys[:n.value], ent[:n.value], arena[:nb.value]


class TransactionValidator:
    """Batch counterpart of the reference's TransactionValidator for the UTXO-context rules."""

    def __init__(self, ctx, params=None):
        self.ctx = ctx
        self._lib = ctx._lib
        self.params = params or Params()

    def validate_populated_transactions(self, batch, pov_daa_score, flags=FLAGS_FULL, host_vm=False):
        """batch.entries must hold the populated UtxoEntry of every input. Returns RESULT_DTYPE[n_txs].
        host_vm=True additionally sends every KGV_TX_NEEDS_HOST_VM transaction through the host script engine."""
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        cb = _c_batch(batch, with_entries=True)
        self.ctx._check(self._lib.kgv_validate_populated(self.ctx._h, ctypes.byref(cb), int(pov_daa_score), int(flags), ctypes.byref(self.params), res.ctypes.data))
        if host_vm:
            self.check_scripts_host(batch, res)
        return res

    def check_scripts_host(self, batch, results):
        """check_scripts with the full host engine (GPU-verified signatures) for every tx whose status is NEEDS_HOST_VM; updates `results` in place."""
        idx = np.nonzero(results["status"] == TX_NEEDS_HOST_VM)[0].astype(np.uint32)
        if len(idx) == 0:
            return results
        out = np.zeros(len(idx), dtype=RESULT_DTYPE)
        cb = _c_batch(batch, with_entries=True)
        self.ctx._check(self._lib.kgv_check_scripts_host(self.ctx._h, ctypes.byref(cb), idx.ctypes.data, len(idx), out.ctypes.data))
        fees = results["fee"][idx]
        results[idx] = out
        results["fee"][idx] = fees
        return results

    def check_scripts(self, batch, results):
        """check_scripts with the full script engine ON THE GPU (kgv_check_scripts) for every tx whose status is NEEDS_HOST_VM; the same
        results as check_scripts_host.  Updates `results` in place (the fee stays)."""
        idx = np.nonzero(results["status"] == TX_NEEDS_HOST_VM)[0].astype(np.uint32)
        if len(idx) == 0:
            return results
        out = np.zeros(len(idx), dtype=RESULT_DTYPE)
        cb = _c_batch(batch, with_entries=True)
        self.ctx._check(self._lib.kgv_check_scripts(self.ctx._h, ctypes.byref(cb), idx.ctypes.data, len(idx), out.ctypes.data))
        fees = results["fee"][idx]
        results[idx] = out
        results["fee"][idx] = fees
        return results

    def validate_mempool_transactions_in_parallel(self, utxo_set, batch, virtual_daa_score, flags=FLAGS_FULL):
        """consensus/src/pipeline/virtual_processor/processor.rs:853-878: the same UTXO-context validation run for a batch of
        mempool transactions against the virtual UTXO set; unlike the block path the per-transaction outcome is RETURNED
        (Vec<TxResult<()>>), not filtered: status / script_err / fail_input say why, `fee` feeds the host-side feerate check
        (tx_validation_in_utxo_context.rs:63-73, f64, stays on the host).  Partially populated transactions (orphans) show up as
        MISSING_OUTPOINTS.  Below a few hundred signature checks per call the CPU path is faster (DESIGN.md §5).
        validate_mempool_transactions_in_utxo_context is the mempool's own rule set: caller entries first, mass computed, feerate threshold."""
        return self.validate_transactions_in_parallel(utxo_set, batch, virtual_daa_score, flags)

    def validate_mempool_transactions_in_utxo_context(self, utxo_set, batch, virtual_daa_score, feerate_threshold=None, non_contextual_mass=None,
                                                      supplied=None):
        """validate_mempool_transaction_in_utxo_context (utxo_validation.rs:341-397) for a batch, through kgv_validate_mempool_txs.
        supplied: None (every input is looked up in `utxo_set`; batch.entries is NOT read, since build_batch fills it with zero records that
        would pass for present entries) or one bool per input: True keeps batch.entries[i] (e.g. an in-mempool parent's output with
        block_daa_score = UNACCEPTED_DAA_SCORE = 2**64 - 1), False looks the input up.
        feerate_threshold: None, or one float per transaction (NaN: None); non_contextual_mass: one value per transaction, the
        max(compute, transient) mass computed in isolation.  Fee / max(storage mass, non_contextual_mass) <= threshold is FeerateTooLow (13).
        Returns (RESULT_DTYPE[n_txs], storage masses u64[n_txs], every input's final entry ENTRY_DTYPE[n_inputs] (pad_[0] = 1: absent),
        the byte arena the entries' script_off points into)."""
        n, ni = batch.n_txs, batch.n_inputs
        if supplied is not None:
            given = batch.entries.copy()
            given["pad_"][:, 0] = np.where(np.asarray(supplied, dtype=bool), 0, 1)
            batch = TxBatch(batch.txs, batch.inputs, batch.outputs, given, batch.arena)
        cb = _c_batch(batch, with_entries=supplied is not None)
        args = None
        if feerate_threshold is not None:
            args = np.zeros(n, dtype=MEMPOOL_ARGS_DTYPE)
            args["feerate_threshold"] = feerate_threshold
            args["non_contextual_mass"] = 0 if non_contextual_mass is None else non_contextual_mass
        res = np.zeros(n, dtype=RESULT_DTYPE)
        mass = np.zeros(n, dtype=np.uint64)
        ent = np.zeros(max(ni, 1), dtype=ENTRY_DTYPE)
        used = ctypes.c_size_t()
        cap = len(batch.arena) + 128 * ni  # caller scripts come from the arena; a looked-up one usually fits 128 bytes
        for _ in range(2):  # the call reports the size it needs before any signature is verified
            arena = np.zeros(max(cap, 8), dtype=np.uint8)
            rc = self._lib.kgv_validate_mempool_txs(self.ctx._h, utxo_set._h, ctypes.byref(cb), int(virtual_daa_score), ctypes.byref(self.params),
                                                    None if args is None else args.ctypes.data, res.ctypes.data, mass.ctypes.data, ent.ctypes.data,
                                                    arena.ctypes.data, len(arena), ctypes.byref(used))
            if rc != ERR_NOMEM or used.value <= cap:
                break
            cap = used.value
        self.ctx._check(rc)
        return res, mass, ent[:ni], arena[:used.value]

    def validate_txs_in_isolation(self, batch, rules=None, ctx_daa_score=0, ctx_past_median_time=0, finality=True):
        """validate_tx_in_isolation, then (finality=True) the lock-time finality of validate_tx_in_header_context_with_args, for every tx of
        the batch (kgv_validate_txs_in_isolation).  Returns (RESULT_DTYPE[n_txs]: status 0 or 14..31, fail_input for the indexed
        variants; TX_MASSES_DTYPE[n_txs]: calc_non_contextual_masses of every tx)."""
        rules = rules or TxRules()
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        masses = np.zeros(batch.n_txs, dtype=TX_MASSES_DTYPE)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_validate_txs_in_isolation(self.ctx._h, ctypes.byref(cb), ctypes.byref(rules), int(ctx_daa_score), int(ctx_past_median_time),
                                                                0 if finality else ISOLATION_SKIP_FINALITY, res.ctypes.data, masses.ctypes.data))
        return res, masses

    def validate_mempool_transactions_in_parallel_full(self, utxo_set, batch, virtual_daa_score, virtual_past_median_time, rules=None,
                                                       feerate_threshold=None, supplied=None):
        """validate_mempool_transactions_in_parallel (processor.rs:853-878) through kgv_validate_mempool_txs_in_parallel: per tx, the
        isolation rules, lock-time finality, then validate_mempool_transactions_in_utxo_context.  A tx rejected by the first two is never
        looked up and gets storage mass 0.  The feerate divisor uses the non-contextual masses computed on the device.  `supplied` and
        `feerate_threshold` as in validate_mempool_transactions_in_utxo_context.  Returns (RESULT_DTYPE[n_txs], storage masses u64[n_txs],
        TX_MASSES_DTYPE[n_txs], every input's final entry ENTRY_DTYPE[n_inputs], the byte arena of their scripts)."""
        rules = rules or TxRules()
        n, ni = batch.n_txs, batch.n_inputs
        if supplied is not None:
            given = batch.entries.copy()
            given["pad_"][:, 0] = np.where(np.asarray(supplied, dtype=bool), 0, 1)
            batch = TxBatch(batch.txs, batch.inputs, batch.outputs, given, batch.arena)
        cb = _c_batch(batch, with_entries=supplied is not None)
        args = None
        if feerate_threshold is not None:
            args = np.zeros(n, dtype=MEMPOOL_ARGS_DTYPE)
            args["feerate_threshold"] = feerate_threshold
        res = np.zeros(n, dtype=RESULT_DTYPE)
        mass = np.zeros(n, dtype=np.uint64)
        masses = np.zeros(n, dtype=TX_MASSES_DTYPE)
        ent = np.zeros(max(ni, 1), dtype=ENTRY_DTYPE)
        used = ctypes.c_size_t()
        cap = len(batch.arena) + 128 * ni
        for _ in range(2):  # the call reports the size it needs before any signature is verified
            arena = np.zeros(max(cap, 8), dtype=np.uint8)
            rc = self._lib.kgv_validate_mempool_txs_in_parallel(self.ctx._h, utxo_set._h, ctypes.byref(cb), int(virtual_daa_score), int(virtual_past_median_time),
                                                                ctypes.byref(self.params), ctypes.byref(rules), None if args is None else args.ctypes.data,
                                                                res.ctypes.data, mass.ctypes.data, masses.ctypes.data, ent.ctypes.data, arena.ctypes.data,
                                                                len(arena), ctypes.byref(used))
            if rc != ERR_NOMEM or used.value <= cap:
                break
            cap = used.value
        self.ctx._check(rc)
        return res, mass, masses, ent[:ni], arena[:used.value]

    def check_transaction_standard_in_isolation(self, batch, masses, policy=None):
        """check_transaction_standard_in_isolation for every tx (kgv_check_txs_standard_in_isolation); masses: TX_MASSES_DTYPE[n_txs], the
        calculated_non_contextual_masses.  Returns (RESULT_DTYPE[n_txs]: status 0 or 32..38, fail_input the input / output index of the
        indexed variants; u64[n_txs] details: the number each verdict carries)."""
        policy = policy or MempoolPolicy()
        m = np.ascontiguousarray(masses, dtype=TX_MASSES_DTYPE)
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        det = np.zeros(batch.n_txs, dtype=np.uint64)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_check_txs_standard_in_isolation(self.ctx._h, ctypes.byref(cb), ctypes.byref(policy), m.ctypes.data, res.ctypes.data,
                                                                      det.ctypes.data))
        return res, det

    def check_transaction_standard_in_context(self, batch, masses, storage_mass, fee, policy=None):
        """check_transaction_standard_in_context for every tx of a populated batch (kgv_check_txs_standard_in_context): storage_mass is
        tx.mass(), fee the calculated_fee, masses the non-contextual masses.  Returns (RESULT_DTYPE[n_txs]: status 0 or 39..42, fee echoed;
        u64[n_txs] details)."""
        policy = policy or MempoolPolicy()
        m = np.ascontiguousarray(masses, dtype=TX_MASSES_DTYPE)
        sm = np.ascontiguousarray(storage_mass, dtype=np.uint64)
        fe = np.ascontiguousarray(fee, dtype=np.uint64)
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        det = np.zeros(batch.n_txs, dtype=np.uint64)
        cb = _c_batch(batch, with_entries=True)
        self.ctx._check(self._lib.kgv_check_txs_standard_in_context(self.ctx._h, ctypes.byref(cb), ctypes.byref(policy), m.ctypes.data, sm.ctypes.data,
                                                                    fe.ctypes.data, res.ctypes.data, det.ctypes.data))
        return res, det

    def is_transaction_output_dust(self, batch, minimum_relay_transaction_fee=1000):
        """is_transaction_output_dust for every output of the batch (kgv_outputs_dust).  Returns bool[n_outputs]."""
        n = len(batch.outputs)
        out = np.zeros(max(n, 1), dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_outputs_dust(self.ctx._h, ctypes.byref(cb), int(minimum_relay_transaction_fee), out.ctypes.data))
        return out[:n].astype(bool)

    def validate_mempool_transactions_with_policy(self, utxo_set, batch, virtual_daa_score, virtual_past_median_time, policy=None, rules=None,
                                                  feerate_threshold=None, supplied=None):
        """validate_mempool_transactions_in_parallel_full with the standardness policy (kgv_validate_mempool_txs_with_policy): standardness in
        isolation, isolation, finality, UTXO context, scripts, then standardness in context for the txs still Ok.  policy=None is
        accept_non_standard = true.  Returns (RESULT_DTYPE[n_txs], storage masses u64[n_txs], TX_MASSES_DTYPE[n_txs], every input's final
        entry ENTRY_DTYPE[n_inputs], the byte arena of their scripts, u64[n_txs] details)."""
        rules = rules or TxRules()
        n, ni = batch.n_txs, batch.n_inputs
        if supplied is not None:
            given = batch.entries.copy()
            given["pad_"][:, 0] = np.where(np.asarray(supplied, dtype=bool), 0, 1)
            batch = TxBatch(batch.txs, batch.inputs, batch.outputs, given, batch.arena)
        cb = _c_batch(batch, with_entries=supplied is not None)
        args = None
        if feerate_threshold is not None:
            args = np.zeros(n, dtype=MEMPOOL_ARGS_DTYPE)
            args["feerate_threshold"] = feerate_threshold
        res = np.zeros(n, dtype=RESULT_DTYPE)
        mass = np.zeros(n, dtype=np.uint64)
        masses = np.zeros(n, dtype=TX_MASSES_DTYPE)
        det = np.zeros(n, dtype=np.uint64)
        ent = np.zeros(max(ni, 1), dtype=ENTRY_DTYPE)
        used = ctypes.c_size_t()
        cap = len(batch.arena) + 128 * ni
        for _ in range(2):  # the call reports the size it needs before any signature is verified
            arena = np.zeros(max(cap, 8), dtype=np.uint8)
            rc = self._lib.kgv_validate_mempool_txs_with_policy(self.ctx._h, utxo_set._h, ctypes.byref(cb), int(virtual_daa_score), int(virtual_past_median_time),
                                                                ctypes.byref(self.params), ctypes.byref(rules), None if args is None else args.ctypes.data,
                                                                res.ctypes.data, mass.ctypes.data, masses.ctypes.data, ent.ctypes.data, arena.ctypes.data,
                                                                len(arena), ctypes.byref(used), None if policy is None else ctypes.byref(policy),
                                                                det.ctypes.data)
            if rc != ERR_NOMEM or used.value <= cap:
                break
            cap = used.value
        self.ctx._check(rc)
        return res, mass, masses, ent[:ni], arena[:used.value], det

    def validate_transactions_with_muhash_in_parallel(self, utxo_set, batch, pov_daa_score, flags=FLAGS_FULL):
        """utxo_validation.rs:282-309: as validate_transactions_in_parallel, plus the combined MuHash::from_transaction of the
        accepted transactions.  Returns (RESULT_DTYPE[n_txs], MuHash)."""
        from .muhash import MuHash
        res = self.validate_transactions_in_parallel(utxo_set, batch, pov_daa_score, flags)
        return res, MuHash.from_transactions(self.ctx, batch, (res["status"] == 0).astype(np.uint8), pov_daa_score, utxo_set=utxo_set)

    def validate_transactions_in_parallel(self, utxo_set, batch, pov_daa_score, flags=FLAGS_FULL):
        """Populate from the GPU UTXO set, then validate. Returns RESULT_DTYPE[n_txs] (coinbase: status 12)."""
        res = np.zeros(batch.n_txs, dtype=RESULT_DTYPE)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_validate_txs(self.ctx._h, utxo_set._h, ctypes.byref(cb), int(pov_daa_score), int(flags), ctypes.byref(self.params), res.ctypes.data))
        return res


class BodyRules(ctypes.Structure):
    """kgv_body_rules; the defaults are mainnet's (MAINNET_PARAMS)."""
    _fields_ = [("max_block_mass", ctypes.c_uint64), ("max_coinbase_payload_len", ctypes.c_uint64)]

    def __init__(self, max_block_mass=500_000, max_coinbase_payload_len=204):
        super().__init__(max_block_mass, max_coinbase_payload_len)


def block_headers(blocks, expected_subsidy, past_median_time=0):
    """BLOCK_HEADER_CTX_DTYPE[n] from blocks_json.load_blocks_json blocks (hash_merkle_root, daa_score, blue_score).  expected_subsidy and
    past_median_time come from the caller's stores: one value for all blocks, one per block, or expected_subsidy as a function of the
    block's daa_score (calc_block_subsidy)."""
    h = np.zeros(len(blocks), dtype=BLOCK_HEADER_CTX_DTYPE)
    for k, b in enumerate(blocks):
        h[k]["hash_merkle_root"] = np.frombuffer(bytes(b["hash_merkle_root"]), dtype=np.uint8)
        h[k]["daa_score"], h[k]["blue_score"] = b["daa_score"], b["blue_score"]
    h["expected_subsidy"] = [expected_subsidy(b["daa_score"]) for b in blocks] if callable(expected_subsidy) else expected_subsidy
    h["past_median_time"] = past_median_time
    return h


class BlockBodyProcessor:
    """Batch counterpart of the reference's BlockBodyProcessor: every rule of validate_body_in_isolation and validate_body_in_context
    (but check_parent_bodies_exist, a statuses-store query) for a window of blocks in one kgv_validate_block_bodies call."""

    def __init__(self, ctx, rules=None, body_rules=None):
        self.ctx = ctx
        self._lib = ctx._lib
        self.rules = rules or TxRules()
        self.body_rules = body_rules or BodyRules()

    def validate_bodies(self, batch, block_first_tx, headers, isolation_only=False):
        """batch: the transactions of all blocks, block b = txs [block_first_tx[b], block_first_tx[b+1]); headers: BLOCK_HEADER_CTX_DTYPE
        per block.  Returns (BODY_RESULT_DTYPE[n_blocks]: the first failing rule of each block, see BODY_STATUS and include/kgv.h;
        BLOCK_MASSES_DTYPE[n_blocks]: the block's Mass, zeros unless Ok; (n_blocks, 32) uint8: the computed hash merkle roots)."""
        f = np.ascontiguousarray(block_first_tx, dtype=np.uint32)
        h = np.ascontiguousarray(headers, dtype=BLOCK_HEADER_CTX_DTYPE)
        n = len(f) - 1
        if len(h) != n:
            raise ValueError("one header record per block")
        res = np.zeros(n, dtype=BODY_RESULT_DTYPE)
        masses = np.zeros(n, dtype=BLOCK_MASSES_DTYPE)
        roots = np.zeros((n, 32), dtype=np.uint8)
        cb = _c_batch(batch, with_entries=False)
        self.ctx._check(self._lib.kgv_validate_block_bodies(self.ctx._h, ctypes.byref(cb), f.ctypes.data, n, h.ctypes.data, ctypes.byref(self.rules),
                                                            ctypes.byref(self.body_rules), BODY_ISOLATION_ONLY if isolation_only else 0,
                                                            res.ctypes.data, masses.ctypes.data, roots.ctypes.data))
        return res, masses, roots

    def validate_blocks(self, blocks, expected_subsidy, past_median_time=0, isolation_only=False):
        """the window form over blocks_json.load_blocks_json blocks: builds the batch and the header records, then validate_bodies"""
        from .txbatch import build_batch
        first = np.cumsum([0] + [len(b["transactions"]) for b in blocks]).astype(np.uint32)
        batch = build_batch([t for b in blocks for t in b["transactions"]])
        return self.validate_bodies(batch, first, block_headers(blocks, expected_subsidy, past_median_time), isolation_only)

    def validate_body_in_isolation(self, block):
        """validate_body_in_isolation for one block: (BODY_RESULT_DTYPE record, BLOCK_MASSES_DTYPE record)"""
        res, masses, _ = self.validate_blocks([block], 0, isolation_only=True)
        return res[0], masses[0]

    def validate_body_in_context(self, block, expected_subsidy, past_median_time=0):
        """validate_body_in_context for one block that passed validate_body_in_isolation: the BODY_RESULT_DTYPE record of the whole order
        (a block failing an isolation rule reports that rule)"""
        return self.validate_blocks([block], expected_subsidy, past_median_time)[0][0]


class SigCache:
    """Device-resident verdict cache (kgv_sigcache): the counterpart of `Cache<SigCacheKey, bool>` (crypto/txscript/src/caches.rs:14-55).
    attach(ctx) makes every validation call of that context consult and fill it."""

    def __init__(self, ctx, capacity=10_000):
        self.ctx = ctx
        h = ctypes.c_void_p()
        ctx._check(ctx._lib.kgv_sigcache_create(ctx._h, int(capacity), ctypes.byref(h)))
        self._h = h

    def attach(self, ctx=None):
        c = ctx or self.ctx
        c._check(c._lib.kgv_set_sigcache(c._h, self._h))

    def detach(self, ctx=None):
        c = ctx or self.ctx
        c._check(c._lib.kgv_set_sigcache(c._h, None))

    def clear(self):
        self.ctx._check(self.ctx._lib.kgv_sigcache_clear(self.ctx._h, self._h))

    def counters(self):
        v = [ctypes.c_uint64() for _ in range(4)]
        self.ctx._check(self.ctx._lib.kgv_sigcache_counters(self.ctx._h, self._h, *[ctypes.byref(x) for x in v]))
        return dict(zip(("hits", "inserts", "lookups", "evictions"), (int(x.value) for x in v)))

    def close(self):
        if self._h:
            self.detach()
            self.ctx._lib.kgv_sigcache_destroy(self._h)
            self._h = None


class KeyCache:
    """A device cache of prepared public keys (kgv_keycache): comb-form key records kept across verify launches, so a key met before runs
    the joint comb ladder in launches of any size.  Capacities are in keys per kind (about 8.4 KB each).  Created on; detach() / attach()
    turn this context's lookups off and on (records kept); verdicts never change.  on(ctx) shares the cache with another context of the
    device."""

    _NAMES = ("lookups", "hits", "inserts", "evictions")

    def __init__(self, ctx, schnorr_keys=1 << 12, ecdsa_keys=1 << 10):
        self.ctx = ctx
        ctx._check(ctx._lib.kgv_keycache_create(ctx._h, int(schnorr_keys), int(ecdsa_keys)))
        self._open = True

    def on(self, ctx):
        """The same cache attached to `ctx`, another context of its device (kgv_keycache_share), as a handle of its own: its attach() /
        detach() switch ctx's lookups, its close() detaches ctx.  The records live until every handle is closed (or its context destroyed),
        in any order."""
        ctx._check(ctx._lib.kgv_keycache_share(ctx._h, self.ctx._h))
        v = KeyCache.__new__(KeyCache)
        v.ctx, v._open = ctx, True
        return v

    def attach(self):
        self.ctx._check(self.ctx._lib.kgv_set_keycache(self.ctx._h, 1))

    def detach(self):
        self.ctx._check(self.ctx._lib.kgv_set_keycache(self.ctx._h, 0))

    def clear(self):
        self.ctx._check(self.ctx._lib.kgv_keycache_clear(self.ctx._h))

    def counters(self, ecdsa=False):
        v = [int(self.ctx._lib.kgv_keycache_counter(self.ctx._h, int(bool(ecdsa)), k)) for k in range(4)]
        if any(x == 2**64 - 1 for x in v):
            self.ctx._check(-2)  # KGV_ERR_CUDA, with the context's message
        return dict(zip(self._NAMES, v))

    def close(self):
        if self._open:
            self._open = False
            self.ctx._check(self.ctx._lib.kgv_keycache_destroy(self.ctx._h))
