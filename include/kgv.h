/*
 * kgv.h — C ABI of the H100 transaction-validation library (libkgv.so).
 *
 * "kgv" = Kaspa GPU Validator.  This is the drop-in boundary for the hot path named by
 * BASELINE.json: batched secp256k1 Schnorr/ECDSA verification, sighash / tx-id hashing, the
 * UTXO table and the fused per-transaction validation that rusty-kaspa fans out over rayon in
 *   consensus/src/pipeline/virtual_processor/utxo_validation.rs:262-309
 *   consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs:34-61,157-196
 *   crypto/txscript/src/lib.rs:574-643
 * The reference has no FFI layer for this path (SURVEY.md §8b): these entry points are what a
 * Rust shim (`extern "C"` block, shown in INTEGRATION.md) binds to stand behind the reference's
 * own TransactionValidator / SigCache / UtxoView surface.
 *
 * Conventions
 *   - plain pointers and sizes only; caller owns every buffer; the library never keeps a host
 *     pointer past the call.
 *   - every data pointer may be a HOST pointer (pageable or pinned) or a DEVICE pointer on the
 *     context's device; the library detects which (cudaPointerGetAttributes), array by array.
 *     A host input is copied in; a device input is read where it is.  A host output is
 *     written through a device copy that comes back before the call returns; a device output
 *     is written in place.  The call synchronises once at its end when some output is host
 *     memory; with device outputs only, the work is enqueued on the context's stream and the
 *     call returns without synchronising (use kgv_synchronize or your own stream sync).
 *     The arrays of a kgv_tx_batch are all host or all device pointers (KGV_ERR_ARG
 *     otherwise).  Each call states which of its other arrays must share one kind
 *     (KGV_ERR_ARG otherwise), which may each be of either kind, and which must be host
 *     memory or device memory.  The parameter structs (kgv_params, kgv_tx_rules, kgv_body_rules,
 *     kgv_mempool_policy, kgv_header_rules), the block and group offsets the library reads to
 *     plan a call, and the scalar results (counts, stats, epochs) are host memory: a device
 *     pointer there gives KGV_ERR_ARG, with kgv_last_error naming the call and the argument.
 *   - return value: 0 = ok, negative = argument / CUDA / NCCL failure (kgv_last_error explains).
 *     An invalid signature is NEVER an error return: verdicts are per-item status bytes.
 *   - there is no CPU fallback: without a usable CUDA device kgv_create fails.
 *   - results are deterministic and independent of batch split or GPU count.
 *   - a context serialises its calls with an internal mutex; use one context per thread for
 *     concurrency.  A UTXO table (plain or a view) may be used from every context of its
 *     device at once, under a reader/writer lock per table (Threading, next to the views).
 */
#ifndef KGV_H
#define KGV_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGV_OK 0
#define KGV_ERR_ARG (-1)
#define KGV_ERR_CUDA (-2)
#define KGV_ERR_NOMEM (-3)
#define KGV_ERR_NCCL (-4)
#define KGV_ERR_LIMIT (-5) /* an internal iteration cap was hit (kgv_check_scripts_host); kgv_last_error says which */

/* Per-signature verdicts.  The reference distinguishes these cases
 * (crypto/txscript/src/lib.rs:582-583, 593, 618-619, 628; SURVEY.md §0-7):
 *   a malformed key / overflowing ECDSA r|s aborts the script with InvalidSignature,
 *   a well-formed but wrong signature is Ok(false) and (in multisig) the loop moves on. */
#define KGV_SIG_INVALID 0       /* sig.verify(..) -> Err  => Ok(false)                       */
#define KGV_SIG_VALID 1         /* sig.verify(..) -> Ok   => Ok(true)                        */
#define KGV_SIG_PK_PARSE_ERR 2  /* XOnlyPublicKey::from_slice / PublicKey::from_slice failed */
#define KGV_SIG_SIG_PARSE_ERR 3 /* ecdsa::Signature::from_compact failed (r or s >= n)       */

typedef struct kgv_ctx kgv_ctx;

/* One context per device.  Builds the generator window tables (8 MiB, L2 resident) on the GPU. */
int kgv_create(int device, uint32_t flags, kgv_ctx** out);
void kgv_destroy(kgv_ctx* ctx);
/* Run all subsequent work of this context on the given cudaStream_t (NULL = CUDA's default
 * stream, as for any cudaStream_t).  Lets a caller bracket kernels with its own events (bench.py
 * passes torch's stream).  kgv_reset_stream goes back to the context's private stream. */
int kgv_set_stream(kgv_ctx* ctx, void* cuda_stream);
int kgv_reset_stream(kgv_ctx* ctx);
int kgv_synchronize(kgv_ctx* ctx);
const char* kgv_last_error(const kgv_ctx* ctx);
/* Number of kernel launches this context has issued so far (bench.py's gpu_launches). */
uint64_t kgv_launch_count(const kgv_ctx* ctx);

/* Batched BIP-340 Schnorr verification: status[i] = verdict of (pk32[i], msg32[i], sig64[i]).
 * Replaces the per-signature FFI call `sig.verify(&msg,&pk)` of
 * crypto/txscript/src/lib.rs:593 together with the parses at :582-583.
 * SoA layout: pk32 = n*32 bytes (x-only key), msg32 = n*32 bytes, sig64 = n*64 bytes (r||s). */
int kgv_schnorr_verify(kgv_ctx* ctx, const uint8_t* pk32, const uint8_t* msg32, const uint8_t* sig64, size_t n, uint8_t* status);

/* Batched ECDSA verification (compressed 33-byte keys, 64-byte compact signatures), with
 * libsecp256k1 semantics: low-S required, r|s >= n is a parse error.
 * Replaces crypto/txscript/src/lib.rs:618-628. */
int kgv_ecdsa_verify(kgv_ctx* ctx, const uint8_t* pk33, const uint8_t* msg32, const uint8_t* sig64, size_t n, uint8_t* status);

/* Pack verdicts into a validity bitmap: bit i (LSB-first within each byte) = (status[i] == KGV_SIG_VALID).
 * bitmap has (n+7)/8 bytes.  This is the per-shard payload of the multi-GPU all-gather. */
int kgv_status_to_bitmap(kgv_ctx* ctx, const uint8_t* status, size_t n, uint8_t* bitmap);

/* ------------------------------------------------------------------------------------------------
 * Flat SoA transaction batches (little-endian, fixed-size records + one byte arena).
 * Mirror of the reference data model: Transaction consensus/core/src/tx.rs:165-185,
 * TransactionInput :93-101, TransactionOutpoint :72-77, TransactionOutput :121-125, UtxoEntry :49-57,
 * ScriptPublicKey tx/script_public_key.rs:22-25.  Offsets point into `bytes`.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  uint32_t first_input, n_inputs;   /* range in inputs[]  */
  uint32_t first_output, n_outputs; /* range in outputs[] */
  uint64_t lock_time, gas;
  uint64_t mass;                    /* committed storage mass (tx.mass()) */
  uint32_t payload_off, payload_len;
  uint16_t version;
  uint8_t subnetwork_id[20];
  uint8_t flags;                    /* bit 0: coinbase (informational; derived from subnetwork_id) */
  uint8_t pad_;
} kgv_tx; /* 72 bytes */
typedef struct {
  uint8_t prev_txid[32];
  uint32_t prev_index;
  uint32_t sigscript_off, sigscript_len;
  uint8_t sig_op_count;
  uint8_t pad_[3];
  uint64_t sequence;
} kgv_input; /* 56 bytes */
typedef struct {
  uint64_t value;
  uint32_t script_off, script_len;
  uint16_t spk_version;
  uint8_t pad_[6];
} kgv_output; /* 24 bytes */
typedef struct {
  uint64_t amount;
  uint64_t block_daa_score;
  uint32_t script_off, script_len;  /* script_public_key.script */
  uint16_t spk_version;
  uint8_t is_coinbase;
  uint8_t pad_[5];                  /* pad_[0] != 0 in a populated batch marks the entry ABSENT (-> MissingTxOutpoints) */
} kgv_utxo_entry; /* 32 bytes */
typedef struct {
  const kgv_tx* txs; size_t n_txs;
  const kgv_input* inputs; size_t n_inputs;
  const kgv_output* outputs; size_t n_outputs;
  const kgv_utxo_entry* entries; /* one populated entry per input (PopulatedTransaction), or NULL */
  const uint8_t* bytes; size_t n_bytes;
} kgv_tx_batch; /* the arrays are all host pointers or all device pointers (KGV_ERR_ARG otherwise) */

/* Transaction ids / hashes of every tx of the batch: out32 = n_txs * 32 bytes.
 * Replaces consensus/core/src/hashing/tx.rs:16-42 (`hash`, `id`; keyed BLAKE2b). */
int kgv_tx_ids(kgv_ctx* ctx, const kgv_tx_batch* batch, uint8_t* out32);
int kgv_tx_hashes(kgv_ctx* ctx, const kgv_tx_batch* batch, uint8_t* out32);

/* Signature hashes.  One item per signature check: `input` is the ABSOLUTE index into
 * batch->inputs / batch->entries, hash_type one of 01 02 04 81 82 84 (anything else yields an
 * all-0xFF digest, sighash_type.rs:50-56 InvalidSigHashType), ecdsa != 0 adds the
 * SHA-256 wrap.  Replaces calc_schnorr_signature_hash / calc_ecdsa_signature_hash
 * (consensus/core/src/hashing/sighash.rs:238-277); the five per-tx sub-hashes are computed once
 * per transaction (SigHashReusedValues, sighash.rs:14-138). */
typedef struct {
  uint32_t tx;
  uint32_t input;
  uint8_t hash_type;
  uint8_t ecdsa;
  uint8_t pad_[2];
} kgv_sighash_item; /* 12 bytes */
int kgv_sighash(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_sighash_item* items, size_t n_items, uint8_t* out32);

/* ------------------------------------------------------------------------------------------------
 * UTXO-context validation (the rayon fan-out of utxo_validation.rs:262-338 as a batch call)
 * ------------------------------------------------------------------------------------------------ */
/* per-transaction verdicts = TxRuleError classes (consensus/core/src/errors/tx.rs:8-103) reachable from
 * validate_transaction_in_utxo_context (utxo_validation.rs:312-338) */
#define KGV_TX_OK 0
#define KGV_TX_MISSING_OUTPOINTS 1      /* MissingTxOutpoints                */
#define KGV_TX_IMMATURE_COINBASE 2      /* ImmatureCoinbaseSpend             */
#define KGV_TX_INPUT_AMOUNT_OVERFLOW 3  /* InputAmountOverflow               */
#define KGV_TX_INPUT_AMOUNT_TOO_HIGH 4  /* InputAmountTooHigh                */
#define KGV_TX_SPEND_TOO_HIGH 5         /* SpendTooHigh                      */
#define KGV_TX_MASS_INCOMPUTABLE 6      /* MassIncomputable                  */
#define KGV_TX_WRONG_MASS 7             /* WrongMass                         */
#define KGV_TX_SEQUENCE_LOCK 8          /* SequenceLockConditionsAreNotMet   */
#define KGV_TX_SIGNATURE_INVALID 9      /* SignatureInvalid(script_err)      */
#define KGV_TX_SIGNATURE_EMPTY 10       /* SignatureEmpty(script_err)        */
#define KGV_TX_NEEDS_HOST_VM 11         /* an input is not one of the GPU fast-path script classes: the host
                                           script engine must decide this transaction (all context checks passed) */
#define KGV_TX_SKIPPED_COINBASE 12      /* coinbase transactions are skipped (utxo_validation.rs:273) */
#define KGV_TX_FEERATE_TOO_LOW 13       /* FeerateTooLow (kgv_validate_mempool_txs only) */
/* validate_tx_in_isolation (tx_validation_in_isolation.rs:16-26) and the lock-time finality of validate_tx_in_header_context
 * (tx_validation_in_header_context.rs): kgv_validate_txs_in_isolation and kgv_validate_mempool_txs_in_parallel only */
#define KGV_TX_NO_TX_INPUTS 14                         /* NoTxInputs                          */
#define KGV_TX_TOO_MANY_INPUTS 15                      /* TooManyInputs                       */
#define KGV_TX_TOO_BIG_SIGNATURE_SCRIPT 16             /* TooBigSignatureScript(fail_input)   */
#define KGV_TX_TOO_MANY_OUTPUTS 17                     /* TooManyOutputs                      */
#define KGV_TX_TOO_BIG_SCRIPT_PUBLIC_KEY 18            /* TooBigScriptPublicKey(output)       */
#define KGV_TX_COINBASE_HAS_INPUTS 19                  /* CoinbaseHasInputs                   */
#define KGV_TX_COINBASE_NON_ZERO_MASS_COMMITMENT 20    /* CoinbaseNonZeroMassCommitment       */
#define KGV_TX_COINBASE_TOO_MANY_OUTPUTS 21            /* CoinbaseTooManyOutputs              */
#define KGV_TX_COINBASE_SCRIPT_PUBLIC_KEY_TOO_LONG 22  /* CoinbaseScriptPublicKeyTooLong(output) */
#define KGV_TX_TX_OUT_ZERO 23                          /* TxOutZero(output)                   */
#define KGV_TX_TX_OUT_TOO_HIGH 24                      /* TxOutTooHigh(output)                */
#define KGV_TX_OUTPUTS_VALUE_OVERFLOW 25               /* OutputsValueOverflow                */
#define KGV_TX_TOTAL_TX_OUT_TOO_HIGH 26                /* TotalTxOutTooHigh                   */
#define KGV_TX_DUPLICATE_INPUTS 27                     /* TxDuplicateInputs                   */
#define KGV_TX_HAS_GAS 28                              /* TxHasGas                            */
#define KGV_TX_SUBNETWORKS_DISABLED 29                 /* SubnetworksDisabled                 */
#define KGV_TX_UNKNOWN_TX_VERSION 30                   /* UnknownTxVersion                    */
#define KGV_TX_NOT_FINALIZED 31                        /* NotFinalized(fail_input)            */
/* the mempool's standardness policy, NonStandardError (mining/errors/src/mempool.rs:100-135): the kgv_check_txs_standard_* calls and
 * kgv_validate_mempool_txs_with_policy only.  detail = the number the variant carries beyond the index (see kgv_mempool_policy). */
#define KGV_TX_REJECT_VERSION 32                       /* RejectVersion               detail: the version       */
#define KGV_TX_REJECT_COMPUTE_MASS 33                  /* RejectComputeMass           detail: the compute mass  */
#define KGV_TX_REJECT_TRANSIENT_MASS 34                /* RejectTransientMass         detail: the transient mass */
#define KGV_TX_REJECT_SIGNATURE_SCRIPT_SIZE 35         /* RejectSignatureScriptSize(fail_input)  detail: its length */
#define KGV_TX_REJECT_SCRIPT_PUBLIC_KEY_VERSION 36     /* RejectScriptPublicKeyVersion(output)              */
#define KGV_TX_REJECT_OUTPUT_SCRIPT_CLASS 37           /* RejectOutputScriptClass(output)                   */
#define KGV_TX_REJECT_DUST 38                          /* RejectDust(output)          detail: its value         */
#define KGV_TX_REJECT_STORAGE_MASS 39                  /* RejectStorageMass           detail: the storage mass  */
#define KGV_TX_REJECT_INPUT_SCRIPT_CLASS 40            /* RejectInputScriptClass(fail_input)                */
#define KGV_TX_REJECT_SIGNATURE_COUNT 41               /* RejectSignatureCount(fail_input)  detail: num_sig_ops */
#define KGV_TX_REJECT_INSUFFICIENT_FEE 42              /* RejectInsufficientFee       detail: the minimum fee   */
/* script errors = TxScriptError variants the standard classes can produce (crypto/txscript/errors) */
#define KGV_SCRIPT_OK 0
#define KGV_SCRIPT_EVAL_FALSE 1
#define KGV_SCRIPT_NULL_FAIL 2
#define KGV_SCRIPT_INVALID_SIGNATURE 3
#define KGV_SCRIPT_SIG_LENGTH 4
#define KGV_SCRIPT_PUBKEY_FORMAT 5
#define KGV_SCRIPT_INVALID_SIGHASH_TYPE 6
#define KGV_SCRIPT_EXCEEDED_SIGOP_LIMIT 7
#define KGV_SCRIPT_NONSTANDARD 255
/* TxValidationFlags (tx_validation_in_utxo_context.rs:20-31) */
#define KGV_FLAGS_FULL 0
#define KGV_FLAGS_SKIP_SCRIPT_CHECKS 1
#define KGV_FLAGS_SKIP_MASS_CHECK 2
/* extension: run ONLY check_scripts on populated entries (no maturity / amount / mass / sequence-lock rules).
 * Signatures are context free given the spent output (SURVEY.md §0-6: the sighash reads only the entry's
 * script_public_key and amount, sighash.rs:252-255), so a window of future blocks can be script-checked in one
 * large batch before the in-order pass, which then runs with KGV_FLAGS_SKIP_SCRIPT_CHECKS. */
#define KGV_FLAGS_SCRIPTS_ONLY 3

typedef struct {
  uint64_t coinbase_maturity;       /* Params::coinbase_maturity      */
  uint64_t storage_mass_parameter;  /* Params::storage_mass_parameter */
  uint64_t max_sompi;               /* constants::MAX_SOMPI           */
} kgv_params;
typedef struct {
  uint64_t fee;        /* calculated_fee (valid when status == KGV_TX_OK) */
  uint32_t fail_input; /* first failing input (index within the tx) for status 2, 9, 10, 11, 16, 31, 35, 40, 41; the first failing OUTPUT
                          (index within the tx) for status 18, 22, 23, 24, 36, 37, 38 */
  uint8_t status;      /* KGV_TX_*     */
  uint8_t script_err;  /* KGV_SCRIPT_* */
  uint8_t pad_[2];
} kgv_tx_result; /* 16 bytes */

/* validate_populated_transaction_and_get_fee for every tx of a batch whose entries are already
 * populated (batch->entries != NULL) — tx_validation_in_utxo_context.rs:34-61 incl. check_scripts
 * (:157-196) for the standard script classes.  results: n_txs records. */
int kgv_validate_populated(kgv_ctx* ctx, const kgv_tx_batch* batch, uint64_t pov_daa_score, uint32_t flags, const kgv_params* params,
                           kgv_tx_result* results);

/* GPU-resident UTXO set: open-addressed hash table keyed by the 36-byte outpoint (txid || index LE),
 * 128-byte slots (entry + up to 68 script bytes inline, longer scripts in an overflow arena).
 * It plays the role of the base layer of every composed view: DbUtxoSetStore
 * (consensus/src/model/stores/utxo_set.rs:31-44,107-112,143-152) and UtxoCollection
 * (consensus/core/src/utxo/utxo_collection.rs:5,28-32). */
typedef struct kgv_utxo_table kgv_utxo_table;
int kgv_utxo_create(kgv_ctx* ctx, uint64_t capacity_slots /* rounded up to a power of two */, kgv_utxo_table** out);
void kgv_utxo_destroy(kgv_ctx* ctx, kgv_utxo_table* t);
/* UtxoView::get for n outpoints: found[i] in {0,1}; entries[i].script_off = i*script_stride into scripts_out
 * (scripts longer than script_stride are truncated there; script_len is always the true length).  Only the script bytes are
 * written: the rest of each script_stride row keeps what the caller put there, whichever side scripts_out is on (a host scripts_out
 * is uploaded first for that).  Each array on its own side. */
int kgv_utxo_lookup(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* keys36, size_t n, kgv_utxo_entry* entries, uint8_t* scripts_out,
                    uint32_t script_stride, uint8_t* found);
/* write_diff_batch (utxo_set.rs:107-112): delete the removed outpoints, then put the added ones.
 * add_entries[i].script_off/len point into add_bytes.  Keys of one call must be distinct.
 * rem_status[i]: 1 = was present, 0 = absent; add_status[i]: 1 = inserted, 2 = replaced an existing entry. */
int kgv_utxo_apply_diff(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* rem_keys36, size_t n_rem, uint8_t* rem_status,
                        const uint8_t* add_keys36, const kgv_utxo_entry* add_entries, const uint8_t* add_bytes, size_t n_add_bytes, size_t n_add,
                        uint8_t* add_status);
/* number of live entries, and an order-independent digest of the set: the sum modulo 2^256 of the keyed
 * BLAKE2b "MuHashElement" hashes of every (outpoint, entry) (consensus/core/src/muhash.rs:47-59). */
int kgv_utxo_count(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t* count);
int kgv_utxo_digest(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t out32[32]);
/* DbUtxoSetStore::iterator (utxo_set.rs:114-129): every live entry as (key, entry record, script bytes), in the table's (arbitrary) order -
 * what the syncer side of a pruning-point import streams out, and what `virtual.utxo_set := pruning-point utxo_set` copies
 * (consensus/src/pipeline/virtual_processor/processor.rs:1150-1158).  Arrays all host or all device.  With keys36 == NULL only the sizes are
 * returned (*n_out entries, *bytes_out script bytes); arrays smaller than that give KGV_ERR_NOMEM with the sizes still set. */
int kgv_utxo_export(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t* keys36, kgv_utxo_entry* entries, uint8_t* bytes, size_t max_n, size_t bytes_cap, size_t* n_out,
                    size_t* bytes_out);
/* append_imported_pruning_point_utxos (consensus/src/consensus/mod.rs:1070-1083) for one chunk of the imported UTXO set: the entries are
 * written into the table (write_many) and MuHash::from_utxo of every (outpoint, entry), reduced, is combined into the running multiset
 * numerator384 (host value, in / out, 384 little-endian bytes; start from 1).  The caller then compares kgv_muhash_finalize(numerator, 1)
 * with the new pruning point's header.utxo_commitment (processor.rs:1133-1139: ImportedMultisetHashMismatch) and validates the pruning
 * point's own transactions with kgv_validate_txs (:1162-1172).  keys36, entries and bytes may each be host or device memory; an entry
 * whose script range leaves the n_bytes arena is refused (KGV_ERR_ARG) on either side. */
int kgv_utxo_import_chunk(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* keys36, const kgv_utxo_entry* entries, const uint8_t* bytes, size_t n_bytes, size_t n,
                          uint8_t* numerator384);

/* Composed views (consensus/core/src/utxo/utxo_view.rs:22-35 ComposedUtxoView / UtxoViewComposition::compose; UtxoDiff utxo_diff.rs:15-19):
 * a DIFF LAYER on the device.  The returned handle is a kgv_utxo_table that every call accepting a table accepts; it behaves as base ∘ diff:
 *   lookups (kgv_utxo_lookup, the populate step of kgv_validate_txs / kgv_replay_window) probe the layer first - an entry it added is found, an
 *   outpoint it removed is absent - and fall through to `base` otherwise (`base` may itself be a view: views nest like the reference's
 *   utxo_set ∘ accumulated_diff ∘ mergeset_diff, processor.rs:437,527);
 *   writes (kgv_utxo_apply_diff, kgv_utxo_apply_accepted, the in-order pass of kgv_replay_window) go to the layer only: removing an entry that
 *   lives below records a removal marker, removing the layer's own addition cancels it, re-adding a removed outpoint keeps the lower entry hidden.
 * `base` is never modified until kgv_utxo_view_commit folds the layer into it (write_diff_batch, utxo_set.rs:107-112); kgv_utxo_view_discard drops
 * the layer's content (a candidate chain that lost).  Count / digest / MuHash are defined on plain tables only.
 *
 * Threading: a table, plain or a view, may be used from any context of its device, at the same time (a table given to a context of another
 * device: KGV_ERR_ARG with a kgv_last_error message).  Each table has a reader/writer lock, with the semantics of the reference's RwLock
 * around the virtual UTXO set (processor.rs:270-272, 556-564, 853-858), ordered on the GPU by CUDA events:
 *   - a call READS a table when it looks entries up in it: kgv_utxo_lookup, _count, _digest, _export, _stats, kgv_utxo_muhash,
 *     kgv_muhash_txs, the populate step of kgv_validate_txs / kgv_validate_mempool_txs / _in_parallel / _with_policy / kgv_replay_window, and
 *     the layer kgv_utxo_view_commit folds.  Reading a view reads every layer below it.  kgv_replay_muhash / _diffs / _verify_chain read the
 *     layers of the last replay window's table (KGV_ERR_ARG when one was rehashed since);
 *   - a call WRITES a table when it changes its slots, arena, counters, capacity or layout: kgv_utxo_apply_diff, _apply_accepted,
 *     _import_chunk, the in-order pass of kgv_replay_window into it, kgv_utxo_view_commit (writes the base), _view_discard, _rehash,
 *     _set_max_load, the growth inside any write, and kgv_utxo_destroy.  A write excludes the reads and writes of every context;
 *   - a read sees the state the writes enqueued before it started left, never part of a write.  Writes to one table take effect in the order
 *     their calls entered.  Writers are preferred: once a write waits, new reads wait behind it, so a steady stream of mempool calls cannot
 *     starve a commit;
 *   - a call that reads a view and writes its top layer (a replay into the layer) reads the layers below and writes the top, so mempool calls
 *     on the base run beside a replay into a view over it.  Only the commit excludes them.
 * A read does not block the host: its stream waits for the event that ends the last write.  A write waits on the host until the open reads of
 * other contexts have finished enqueuing (the reference's upgrade()), then its stream waits for their events.  A call holds its tables from
 * its first enqueued access to its last, host synchronisations inside it included; a call touching several tables takes them bottom layer
 * first.  Arrays a write gives up (rehash, growth) are freed once that write has completed on the GPU, at the writing context's
 * kgv_synchronize or kgv_destroy; kgv_utxo_destroy frees the rest.  With one context nothing changes but one event record and one stream wait
 * per table and call.  A table must outlive every call on it, from every context.  The partitions of a key cache shared by several contexts
 * (kgv_keycache_share) take the same lock, per verify launch and always after a call's tables (Key cache, Threading). */
int kgv_utxo_view_create(kgv_ctx* ctx, kgv_utxo_table* base, uint64_t capacity_slots, kgv_utxo_table** out);
int kgv_utxo_view_commit(kgv_ctx* ctx, kgv_utxo_table* view);
int kgv_utxo_view_discard(kgv_ctx* ctx, kgv_utxo_table* view);

/* Table maintenance.  An erase leaves a tombstone and a probe for an absent key ends only at an EMPTY slot, so a table that churns for long
 * slows down every lookup that misses and every insert until it is rebuilt; long scripts are appended to the overflow arena and their bytes
 * are only reclaimed by a rebuild.  All three calls work on plain tables and on view layers (a layer alone, never the layers below it). */
typedef struct {
  uint64_t capacity_slots;
  uint64_t live;              /* entries (in a view layer: also its removal markers) */
  uint64_t tombstones;
  uint64_t empty;             /* EMPTY slots */
  uint64_t overflow_used;     /* bytes appended to the long-script arena (8-byte padded) */
  uint64_t overflow_cap;
  uint64_t overflow_live;     /* of those, the bytes the live entries' scripts occupy (= overflow_used right after a rehash) */
  uint64_t insert_failures;   /* entries lost to a full table or arena since the table was created (never reset) */
  uint64_t rehashes;          /* times this handle was rebuilt */
  uint64_t max_displacement;  /* over the entries: (slot - home slot) mod capacity */
  uint64_t sum_displacement;
  uint64_t longest_run;       /* longest circular run of non-EMPTY slots: the probes of the worst lookup that misses */
} kgv_utxo_table_stats; /* 96 bytes */
/* One pass over the slots; synchronises the context's stream. */
int kgv_utxo_stats(kgv_ctx* ctx, kgv_utxo_table* t, kgv_utxo_table_stats* out);
/* Rebuild out of place into capacity_slots (0: the current capacity; else rounded up to a power of two, so the table can grow or shrink):
 * tombstones are dropped and the long-script arena is compacted; entries, count and digest stay as they are, insert_failures too.
 * A capacity below live + 1 gives KGV_ERR_ARG, a failed allocation KGV_ERR_NOMEM; either leaves the table untouched.  The old and the new
 * arrays exist side by side during the call; the old ones are released at the next kgv_synchronize (or when an allocation needs the memory).
 * View layers above the table keep working.  A rehash ends the window kgv_replay_muhash refers to (call that first). */
int kgv_utxo_rehash(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t capacity_slots);
/* Growth policy, off (0) by default.  With 1..900 every call that writes to `t` (kgv_utxo_apply_diff, kgv_utxo_import_chunk,
 * kgv_utxo_apply_accepted, kgv_replay_window, and kgv_utxo_view_commit for the base) first makes room: when its entries would pass
 * max_load_permille of the capacity the table grows to the smallest power of two that keeps them at half that load; when entries plus
 * tombstones would, or the arena cannot take the call's long scripts, it is rehashed at its size.  It never shrinks.  The check keeps an
 * upper bound of the occupied slots on the host and reads the device counters (one synchronisation) only when that bound reaches the
 * threshold.  The byte bound of a batch call assumes its scripts are disjoint ranges of its byte arena.  A failed growth makes the
 * writing call return KGV_ERR_NOMEM before it writes anything. */
int kgv_utxo_set_max_load(kgv_ctx* ctx, kgv_utxo_table* t, uint32_t max_load_permille);

/* validate_transactions_in_parallel (utxo_validation.rs:262-278) against the table: populate every input
 * by table lookup (:319-327), then as kgv_validate_populated.  batch->entries is ignored.
 * Unlike kgv_validate_populated this call never reports KGV_TX_NEEDS_HOST_VM: transactions with non-standard scripts are
 * decided inside the call by the full script engine on the GPU (kgv_check_scripts) on the entries the table returned (the reference accepts ANY
 * transaction whose scripts execute successfully, utxo_validation.rs:282-309). */
int kgv_validate_txs(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t pov_daa_score, uint32_t flags, const kgv_params* params,
                     kgv_tx_result* results);
/* UtxoDiff::add_transaction (utxo_diff.rs:233-247) applied directly to the table for every tx with
 * accept[i] != 0: spent outpoints are erased, outputs inserted with block_daa_score = pov_daa_score and
 * is_coinbase of the tx (tx ids are computed on the device). */
int kgv_utxo_apply_accepted(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, const uint8_t* accept, uint64_t pov_daa_score);

/* validate_mempool_transaction_in_utxo_context (consensus/src/pipeline/virtual_processor/utxo_validation.rs:341-397) for every tx of a
 * batch against the virtual UTXO view `virtual_view` (a table or a composed view):
 *   populate   an input keeps the entry the caller supplies (batch->entries[i] with pad_[0] == 0: e.g. an in-mempool parent's output, whose
 *              block_daa_score is UNACCEPTED_DAA_SCORE = u64::MAX); only the inputs without one are looked up, and every input is tried
 *              (:348-358).  batch->entries may be NULL: everything is looked up.
 *   rules      missing outpoints -> storage mass (MassIncomputable) -> coinbase maturity -> input amounts -> spend -> sequence lock ->
 *              feerate -> scripts.  The committed mass is not checked (SkipMassCheck, :392); the computed one is returned.
 *   feerate    with args[i].feerate_threshold not NaN: fee as f64 / max(storage mass, args[i].non_contextual_mass) as f64 <= threshold is
 *              KGV_TX_FEERATE_TOO_LOW (tx_validation_in_utxo_context.rs:63-73).  It comes before the scripts, so such a transaction's
 *              signatures are never verified nor cached.  A threshold whose divisor is 0 makes the call fail with KGV_ERR_ARG (the reference
 *              asserts it is not zero).  args == NULL: no thresholds.
 * Non-standard scripts are decided inside the call by the device script engine, as in kgv_validate_txs; coinbases give KGV_TX_SKIPPED_COINBASE.
 * results: n_txs records (fee set once the amounts pass); storage_mass: n_txs values (0 when the mass was not reached).
 * entries_out (n_inputs records, may be NULL): every input's final entry - the caller's, the one found, or absent-marked (pad_[0] = 1) when
 * neither - with script_off into scripts_out (scripts_cap bytes).  *scripts_used (may be NULL) receives the bytes those scripts take; when
 * entries_out is given and they exceed scripts_cap the call returns KGV_ERR_NOMEM before any signature is verified, with *scripts_used set
 * (script_off is 32 bits: scripts above 4 GiB in all give KGV_ERR_ARG when entries_out is given).  The entries are written before the script
 * phase runs.  Every data pointer (batch, args, outputs) host or every one device; a mix gives KGV_ERR_ARG. */
typedef struct {
  double feerate_threshold;     /* NaN: None */
  uint64_t non_contextual_mass; /* max(compute mass, transient mass) the caller computed in isolation */
} kgv_mempool_tx_args;          /* 16 bytes */
int kgv_validate_mempool_txs(kgv_ctx* ctx, kgv_utxo_table* virtual_view, const kgv_tx_batch* batch, uint64_t virtual_daa_score, const kgv_params* params,
                             const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_utxo_entry* entries_out,
                             uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used);

/* The per-transaction rules that need no UTXO context: validate_tx_in_isolation (tx_validation_in_isolation.rs:16-26), the lock-time
 * finality of validate_tx_in_header_context_with_args (tx_validation_in_header_context.rs) and calc_non_contextual_masses
 * (consensus/core/src/mass/mod.rs:248-269).  The fields are the reference's Params of the same names (kgv_params is frozen). */
typedef struct {
  uint64_t max_tx_inputs;
  uint64_t max_tx_outputs;
  uint64_t max_signature_script_len;
  uint64_t max_script_public_key_len;
  uint64_t mass_per_tx_byte;
  uint64_t mass_per_script_pub_key_byte;
  uint64_t mass_per_sig_op;
  uint64_t ghostdag_k;                                 /* a coinbase may have ghostdag_k + 2 outputs */
  uint64_t coinbase_payload_script_public_key_max_len;
} kgv_tx_rules; /* 72 bytes */
typedef struct {
  uint64_t compute_mass;   /* NonContextualMasses::compute_mass   */
  uint64_t transient_mass; /* NonContextualMasses::transient_mass */
} kgv_tx_masses; /* 16 bytes */
#define KGV_ISOLATION_SKIP_FINALITY 1u /* run validate_tx_in_isolation alone */

/* validate_tx_in_isolation then validate_tx_in_header_context_with_args(tx, ctx_daa_score, ctx_past_median_time) for every tx of a batch
 * (batch->entries is not read).  The checks run in the reference's order and the first failing one gives the status (KGV_TX_OK or 14..31),
 * with fail_input set for the indexed variants; fee and script_err are 0.  A tx is a coinbase when its subnetwork_id is the coinbase
 * subnetwork id (kgv_tx.flags is not read).  MAX_SOMPI and LOCK_TIME_THRESHOLD are the consensus constants.  Finality: lock_time 0 is
 * final; a lock_time below 500 000 000 000 is compared with ctx_daa_score, any other with ctx_past_median_time; lock_time < that value is
 * final; otherwise the first input whose sequence is not u64::MAX gives KGV_TX_NOT_FINALIZED.  flags: KGV_ISOLATION_SKIP_FINALITY or 0.
 * results: n_txs records.  masses (may be NULL): n_txs calc_non_contextual_masses records, computed for every tx whatever its status, in
 * wrapping u64 arithmetic ((0, 0) for a coinbase).  Every data pointer host or every one device. */
int kgv_validate_txs_in_isolation(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_tx_rules* rules, uint64_t ctx_daa_score, uint64_t ctx_past_median_time,
                                  uint32_t flags, kgv_tx_result* results, kgv_tx_masses* masses);

/* validate_mempool_transactions_in_parallel (processor.rs:853-878): per tx, what validate_mempool_transaction_impl (:823-839) does -
 * kgv_validate_txs_in_isolation's checks with (virtual_daa_score, virtual_past_median_time), then kgv_validate_mempool_txs.  A tx that
 * fails isolation or finality gets that status, storage_mass 0, and is never looked up: its entries_out rows are the caller's entries
 * where batch->entries supplies them and absent-marked otherwise; it reaches neither the context rules nor the scripts nor the SigCache.
 * The feerate divisor is max(storage mass, compute mass, transient mass) with the masses computed here (what the mempool stores in
 * calculated_non_contextual_masses before it validates): args[i].non_contextual_mass is IGNORED, only feerate_threshold is read.
 * masses (may be NULL): n_txs records as in kgv_validate_txs_in_isolation.  Everything else as kgv_validate_mempool_txs. */
int kgv_validate_mempool_txs_in_parallel(kgv_ctx* ctx, kgv_utxo_table* virtual_view, const kgv_tx_batch* batch, uint64_t virtual_daa_score,
                                         uint64_t virtual_past_median_time, const kgv_params* params, const kgv_tx_rules* rules,
                                         const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_tx_masses* masses,
                                         kgv_utxo_entry* entries_out, uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used);

/* The mempool's standardness policy (mining/src/mempool/check_transaction_standard.rs), which a node that does not relay non-standard
 * transactions (Config::accept_non_standard = false) applies to every transaction it admits.  The limits are the reference's constants:
 * MAXIMUM_STANDARD_TRANSACTION_MASS 100 000, MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE 1 650, MAX_STANDARD_P2SH_SIG_OPS 15 (:13-38).
 * The fields are mining/src/mempool/config.rs's of the same names; the defaults there are 1 000 sompi/kg and TX_VERSION (0) for both versions.
 * detail (may be NULL, n_txs values): the number the verdict carries beyond its index (KGV_TX_REJECT_* above), 0 for any other status. */
typedef struct {
  uint64_t minimum_relay_transaction_fee;          /* sompi per 1 000 grams of mass */
  uint16_t minimum_standard_transaction_version;
  uint16_t maximum_standard_transaction_version;
  uint8_t pad_[4];
} kgv_mempool_policy; /* 16 bytes */

/* check_transaction_standard_in_isolation (:41-105) for every tx: version range, compute mass, transient mass (masses: the caller's
 * calculated_non_contextual_masses, n_txs records), the first input whose signature script exceeds 1 650 bytes, then the outputs in order
 * - per output its spk version (> 0), its ScriptClass (script_class.rs:39-82: NonStandard) and dust, the first failing check of the first
 * failing output.  results: n_txs records, status KGV_TX_OK or 32..38, fee 0.  Every data pointer host or every one device. */
int kgv_check_txs_standard_in_isolation(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_mempool_policy* policy, const kgv_tx_masses* masses,
                                        kgv_tx_result* results, uint64_t* detail);
/* check_transaction_standard_in_context (:172-211) for every tx of a batch whose entries are populated (batch->entries required):
 * storage_mass[i] > 100 000 (tx.mass(), the storage mass the UTXO-context validation computed), then per input the entry's ScriptClass
 * (NonStandard) and, for a P2SH entry, get_sig_op_count_upper_bound(signature script) > 15 (crypto/txscript/src/lib.rs:176-226); INSIDE
 * that loop fee[i] (calculated_fee) < minimum_required_transaction_relay_fee(masses[i].compute_mass) (:215-231) is RejectInsufficientFee.
 * The fee check does not depend on the input, so the order is: storage mass, input 0, the fee, inputs 1..; a tx without inputs never has
 * its fee checked.  Where the reference's sig-op count panics (OP_16 before a multisig opcode: to_small_int's range excludes OP_16) the
 * count takes 16, the value OP_16 stands for.  results: status KGV_TX_OK or 39..42, fee = fee[i].  A relay fee with mass * fee above
 * u64::MAX for a tx whose fee check is reached (the reference's overflow check panics) makes the call return KGV_ERR_ARG. */
int kgv_check_txs_standard_in_context(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_mempool_policy* policy, const kgv_tx_masses* masses,
                                      const uint64_t* storage_mass, const uint64_t* fee, kgv_tx_result* results, uint64_t* detail);
/* is_transaction_output_dust (:116-163; MiningManager::is_transaction_output_dust, mining/src/manager.rs:819) for every output of the batch:
 * is_dust[o] = 1 when the script is unspendable (a parse error anywhere, or OP_RETURN first: crypto/txscript/src/lib.rs:231-233) or
 * value * 1000 / (3 * (8 + 2 + 8 + script_len + 148)) < minimum_relay_transaction_fee, computed exactly in 128 bits.  Scripts of any
 * length; the version and class are not read.  is_dust: n_outputs bytes, host or device as the batch. */
int kgv_outputs_dust(kgv_ctx* ctx, const kgv_tx_batch* batch, uint64_t minimum_relay_transaction_fee, uint8_t* is_dust);
/* kgv_validate_mempool_txs_in_parallel with the standardness policy, in the mempool's admission order
 * (mining/src/mempool/validate_and_insert_transaction.rs:20-33, 142-159):
 *   1. standardness in isolation, on the non-contextual masses the call computes;
 *   2. isolation and finality;  3. UTXO context and feerate;  4. scripts;
 *   5. standardness in context, for the transactions whose status is still KGV_TX_OK (storage mass and fee of this call).
 * A tx rejected in step 1 is never looked up, verified or cached, as an isolation failure (its entries_out rows likewise); one rejected in
 * step 5 has had its signatures verified (and cached).  policy == NULL is accept_non_standard = true: the call is then exactly
 * kgv_validate_mempool_txs_in_parallel.  detail (may be NULL): as above.  The relay-fee overflow of kgv_check_txs_standard_in_context can
 * only occur when minimum_relay_transaction_fee > u64::MAX / 100 000; only then does a device-pointer call synchronise once more. */
int kgv_validate_mempool_txs_with_policy(kgv_ctx* ctx, kgv_utxo_table* virtual_view, const kgv_tx_batch* batch, uint64_t virtual_daa_score,
                                         uint64_t virtual_past_median_time, const kgv_params* params, const kgv_tx_rules* rules,
                                         const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_tx_masses* masses,
                                         kgv_utxo_entry* entries_out, uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used,
                                         const kgv_mempool_policy* policy, uint64_t* detail);

/* ------------------------------------------------------------------------------------------------
 * SigCache: Cache<SigCacheKey, bool> (crypto/txscript/src/caches.rs:14-55; consulted at crypto/txscript/src/lib.rs:589-603, 624-638;
 * created with 10 000 entries and shared by every clone of the TransactionValidator, transaction_validator/mod.rs:48).
 * A device-resident, bounded table of verdicts keyed by BLAKE2b-256(kind || signature || public key || message).  Attached to a context
 * (kgv_set_sigcache; several contexts of one device may share one cache, as the clones share the Arc), it is consulted by the script
 * phase of kgv_validate_populated / kgv_validate_txs / kgv_replay_window: pairs seen before are answered from the table, only the
 * misses reach the verification kernels, and their verdicts (true AND false; never parse errors, which the reference raises before its
 * cache) are remembered.  Full neighbourhoods evict a pseudo-random entry (caches.rs:49-51).  Results never change, only speed:
 * block-template building and block validation re-meet what the mempool verified (processor.rs:853-914).
 * capacity is rounded up to a power of two.  counters: hits = get_counts, inserts = insert_counts (caches.rs:57-93).
 * ------------------------------------------------------------------------------------------------ */
typedef struct kgv_sigcache kgv_sigcache;
int kgv_sigcache_create(kgv_ctx* ctx, uint64_t capacity, kgv_sigcache** out);
void kgv_sigcache_destroy(kgv_sigcache* cache);
int kgv_sigcache_clear(kgv_ctx* ctx, kgv_sigcache* cache);
int kgv_sigcache_counters(kgv_ctx* ctx, kgv_sigcache* cache, uint64_t* hits, uint64_t* inserts, uint64_t* lookups, uint64_t* evictions);
int kgv_set_sigcache(kgv_ctx* ctx, kgv_sigcache* cache /* NULL: detach */);

/* ------------------------------------------------------------------------------------------------
 * Key cache: prepared public keys kept across verify launches.  The reference has no counterpart: libsecp256k1 lifts the key and builds
 * its tables on every secp256k1_schnorrsig_verify / secp256k1_ecdsa_verify, and so does every verify launch here without it (per-launch
 * records only in launches of more items than the device's resident threads whose keys repeat).
 * An opt-in, device-resident table of comb-form key records (8 320 bytes each, about 8.4 KB per key with its slot: 2^16 keys take about
 * 550 MB), off by default, that the contexts of one device can share.  While it is on for a context, every verify launch of that context
 * (the verify entry points, validation, mempool validation, replay windows, the device script engine, the SigCache's misses) looks its
 * keys up: a stored key's signatures run the 30-doubling joint comb ladder from the stored record whatever the launch's size, the other
 * keys are verified as without the cache and stored for the next launch of any context sharing it (a launch of at most one item per
 * resident thread stores them after its verification, off the call's path; a larger one stores them first when the per-launch rule would
 * prepare records and the cache holds them all, else it runs as without the cache).  Verdicts never depend on it.  Where it loses: a
 * launch that stores many new keys (cold large launches build a full record per key, even for keys used a few times), and the call right
 * after one that stored keys (it waits for that insert); DESIGN.md §5 has the numbers.
 * - kgv_keycache_create creates a cache and attaches it to the context, on: one partition per item kind with its own capacity in keys (0:
 *   that kind is not cached), Schnorr keyed by x, ECDSA by tag || x (02 and 03 of one x are two keys).  Both 0, one above
 *   KGV_KEYCACHE_MAX_KEYS, or a context that has a cache is KGV_ERR_ARG; memory that cannot be allocated KGV_ERR_NOMEM.
 * - kgv_keycache_share attaches the cache `holder` has to `ctx` as well, on for ctx: one cache per device, so a key the mempool context met
 *   is stored for the block and template contexts too, and the records exist once.  KGV_ERR_ARG (naming the call) when holder has no cache,
 *   ctx already has one, ctx == holder, or the two contexts are on different devices.  Under sharding each rank's context has its own cache.
 * - Eight-way sets; a full set replaces its least recently used key, never one that a launch still running reads.
 * - kgv_set_keycache turns the context's lookups off (0) and on again, keeping the records; another context attached to the same cache
 *   keeps its own setting (a mempool context keeps it on while an IBD context turns it off).
 * - kgv_keycache_clear empties both partitions of the cache and zeroes their counters, for every context attached to it.
 * - kgv_keycache_destroy detaches the context (KGV_OK without a cache; kgv_destroy does the same) after waiting for its own launches and
 *   inserts; the records are freed when the last attached context detaches, the creator included, in any order.
 * - kgv_keycache_counter: a counter of the partition ecdsa selects, shared by every attached context (0 without a cache, that partition, or
 *   with a bad argument; UINT64_MAX when the device fails): KGV_KEYCACHE_LOOKUPS items looked up, KGV_KEYCACHE_HITS items verified from a
 *   stored record (a large launch the cache does not take counts its lookups, no hits), KGV_KEYCACHE_INSERTS keys stored,
 *   KGV_KEYCACHE_EVICTIONS stored keys replaced; stored keys = inserts - evictions.  It covers the launches of every attached context
 *   enqueued before the call.
 * Threading: the contexts attached to one cache may run at the same time, each from its own thread.  Each partition has the reader/writer
 * lock of the UTXO tables (Threading, next to the views), ordered on the GPU by CUDA events: a verify launch READS the partition from its
 * lookup to the end of its stored-record launch; storing keys, the clear and the counter reads WRITE it.  A launch's stamps and counters
 * are atomics that concurrent readers share, so two contexts' lookups run side by side; an insert waits on the GPU for the reads enqueued
 * before it and excludes every other access while it runs, so no launch of any context reads a record that is being rewritten.  A
 * registration covers one launch's enqueue, taken after any UTXO table lock of its call and holding no other lock, so a write waits on the
 * host only for other contexts to finish enqueuing a launch, never for a whole call or its host synchronisations.  With one context
 * nothing changes but the lock's event records and stream waits: one of each per lookup, one record and two waits per insert.
 * ------------------------------------------------------------------------------------------------ */
#define KGV_KEYCACHE_MAX_KEYS (1ull << 20) /* per kind: about 8.8 GB of records */
enum { KGV_KEYCACHE_LOOKUPS = 0, KGV_KEYCACHE_HITS = 1, KGV_KEYCACHE_INSERTS = 2, KGV_KEYCACHE_EVICTIONS = 3 };
int kgv_keycache_create(kgv_ctx* ctx, uint64_t schnorr_keys, uint64_t ecdsa_keys);
int kgv_keycache_share(kgv_ctx* ctx, kgv_ctx* holder);
int kgv_keycache_destroy(kgv_ctx* ctx);
int kgv_keycache_clear(kgv_ctx* ctx);
uint64_t kgv_keycache_counter(kgv_ctx* ctx, int ecdsa, int which);
int kgv_set_keycache(kgv_ctx* ctx, int enabled);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU (SURVEY.md §8b kgv_shard_allgather, §8e): signature batches shard across GPUs as contiguous ranges, one context (and
 * normally one process) per GPU; the only exchange step of the path is "every rank ends up with every shard's verdicts".
 * The reference has no counterpart (rayon on one host, utxo_validation.rs:269-277).
 *
 * A communicator binds a context to its place among n_ranks and offers two transports:
 *   NCCL  (id != NULL): kgv_shard_allgather = ncclAllGather on the context's stream.  libnccl.so.2 is resolved at run time;
 *         KGV_ERR_NCCL if it is missing.  The 128-byte id comes from kgv_comm_unique_id on rank 0 and reaches the other ranks
 *         through whatever the host uses (MPI, TCP, torch.distributed).
 *   peer  (slice_capacity_bytes != 0): every rank owns receive buffers its peers map (kgv_comm_export -> host exchanges the
 *         handles -> kgv_comm_import; or kgv_comm_connect_local for several contexts of ONE process).  kgv_shard_publish_* is the
 *         PRODUCING kernel writing its shard straight into every peer over NVLink and raising an epoch flag there;
 *         kgv_shard_wait waits on local flags.  No collective, no host rendezvous.  Every rank must publish the same sequence
 *         of epochs and wait for epoch e before publishing e + 1.
 * ------------------------------------------------------------------------------------------------ */
typedef struct kgv_comm kgv_comm;
#define KGV_COMM_ID_BYTES 128
#define KGV_COMM_HANDLE_BYTES 64
int kgv_comm_unique_id(uint8_t id[KGV_COMM_ID_BYTES]);
int kgv_comm_create(kgv_ctx* ctx, int n_ranks, int rank, const uint8_t* id /* NULL: no NCCL */, size_t slice_capacity_bytes /* 0: no peer buffers */,
                    kgv_comm** out);
void kgv_comm_destroy(kgv_comm* comm);
int kgv_comm_export(kgv_comm* comm, uint8_t handle[KGV_COMM_HANDLE_BYTES]);
int kgv_comm_import(kgv_comm* comm, const uint8_t* handles /* n_ranks * KGV_COMM_HANDLE_BYTES, indexed by rank */);
int kgv_comm_connect_local(kgv_comm* const* comms, int n /* comms[i] has rank i */);
/* all_shards[r * nbytes_per_rank ..) = rank r's local_shard, on every rank (device pointers; in place allowed as in NCCL). */
int kgv_shard_allgather(kgv_ctx* ctx, kgv_comm* comm, const uint8_t* local_shard, size_t nbytes_per_rank, uint8_t* all_shards);
/* peer transport.  publish_bitmap: kgv_status_to_bitmap fused with the transfer (status: n device bytes; the shard is 4*ceil(n/32) bytes);
 * publish_bytes: a raw device array.  *epoch_out names the exchange.  wait: enqueue the wait for `epoch` and (all_shards != NULL)
 * copy the n_ranks received shards, nbytes_per_rank each, into one contiguous device array. */
int kgv_shard_publish_bitmap(kgv_ctx* ctx, kgv_comm* comm, const uint8_t* status, size_t n, uint64_t* epoch_out);
int kgv_shard_publish_bytes(kgv_ctx* ctx, kgv_comm* comm, const uint8_t* src, size_t nbytes, uint64_t* epoch_out);
int kgv_shard_wait(kgv_ctx* ctx, kgv_comm* comm, uint64_t epoch, size_t nbytes_per_rank, uint8_t* all_shards);
/* Shard the signature checks of this context's validation calls (kgv_replay_window, kgv_validate_*) over the communicator's
 * ranks (BASELINE configs[4]): every rank runs the same call on the same batch against its own replica of the UTXO table;
 * the candidate (signature, key) pairs are split into n_ranks contiguous ranges, each rank verifies one range and the verdicts
 * are exchanged (peer transport if connected, else NCCL) before the scripts are resolved - identically on every rank.
 * comm == NULL switches sharding off. */
int kgv_set_sharding(kgv_ctx* ctx, kgv_comm* comm);

/* ------------------------------------------------------------------------------------------------
 * DAG replay: calculate_utxo_state / verify_expected_utxo_state (utxo_validation.rs:110-173,182-228) for a WINDOW of
 * blocks as one device-resident call; the loop simpa times (simpa/src/main.rs:454-460).
 *
 * The batch holds the transactions of all blocks of the window, block after block; blocks[] (a HOST array) tiles it.
 * Transaction 0 of every block is its coinbase and is skipped by position (utxo_validation.rs:273).  Semantics are those
 * of processing the blocks one by one, in order, against the table:
 *     validate_transactions_in_parallel(block txs, table, pov_daa_score, Full | SkipScriptChecks)
 *     UtxoDiff::add_transaction for every accepted transaction (and for the coinbase when ACCEPT_COINBASE is set)
 * but every signature of the window is verified in one batch up front (signatures are context free given the spent
 * output, SURVEY.md §0-6) and the in-order pass is a single persistent kernel.
 * All merged blocks of one chain block carry that chain block's pov_daa_score (:124-151).
 * ------------------------------------------------------------------------------------------------ */
#define KGV_REPLAY_ACCEPT_COINBASE 1u /* the block is the selected parent of its chain block: its coinbase is accepted (:116-121) */
#define KGV_REPLAY_SKIP_SCRIPTS 2u    /* TxValidationFlags::SkipScriptChecks for this block (selected parent, :138-140) */
#define KGV_REPLAY_VERIFY_ONLY 4u     /* validate against the current view, apply nothing (verify_expected_utxo_state, :219-225) */
typedef struct {
  uint32_t first_tx, n_txs; /* range of batch->txs; tx first_tx is the block's coinbase */
  uint64_t pov_daa_score;
  uint32_t flags;           /* KGV_REPLAY_* */
  uint32_t pad_;
} kgv_replay_block; /* 24 bytes */
typedef struct {
  uint64_t n_accepted;   /* accepted non-coinbase transactions */
  uint64_t n_sig_checks; /* candidate (signature, key) pairs verified in the pre-check */
  uint64_t n_host_vm;    /* transactions the fast path declined, decided by the full script engine */
  float pre_check_ms;    /* device time of the batched script pre-check (tx ids, window map, populate, sighash, verify, resolve) */
  float in_order_ms;     /* device time from the end of the pre-check to the end of the finishing passes (slot map, static rules, walk,
                            verdicts, table updates, results) */
} kgv_replay_stats;
/* results: n_txs records (host or device memory): the UTXO-context verdict when the context rules fail, else the script
 * verdict (KGV_TX_SKIPPED_COINBASE for coinbases).  accept (may be NULL): n_txs bytes, 1 = folded into the table.
 * stats may be NULL.  results and accept are each on their own side; blocks, params and stats are host memory. */
int kgv_replay_window(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, const kgv_replay_block* blocks, size_t n_blocks,
                      const kgv_params* params, kgv_tx_result* results, uint8_t* accept, kgv_replay_stats* stats);

/* The multiset of what the LAST kgv_replay_window call of this context accepted, per group of blocks: group g = blocks
 * [group_first_block[g], group_first_block[g+1]) of that window (the mergeset of one chain block); values768[g] = (numerator || denominator) of
 * MuHash::from_transaction over the accepted transactions of the group incl. accepted coinbases (utxo_validation.rs:116-121,144; spent entries as
 * found at each block's position).  Must directly follow that kgv_replay_window call (no other batch call in between).
 * With kgv_muhash_prefix_combine and kgv_muhash_finalize_batch this yields every chain block's utxo_commitment of a window (:188-192);
 * kgv_replay_verify_chain (after kgv_validate_block_bodies below) does that and the rest of verify_expected_utxo_state in one call. */
int kgv_replay_muhash(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, uint8_t* values768);
/* The UtxoDiff of every group of blocks of the LAST kgv_replay_window call (ctx.mergeset_diff of calculate_utxo_state, utxo_validation.rs:119,148:
 * what commit_utxo_state stores per chain block and what reorgs read back).  Groups tile the window as in kgv_replay_muhash (group_first_block:
 * a HOST array).  Group g's diff is UtxoDiff::add_transaction (utxo_diff.rs:224-260) of every transaction the window accepted in its blocks, in
 * block order then transaction order (accepted coinbases included, VERIFY_ONLY blocks contribute nothing), with each spent entry as it was found
 * at its block's position.  So an output created and spent inside one group is in neither list, and one created in group g and spent in a later
 * group g' is in g's add (block_daa_score = the accepting block's) and in g''s remove.
 *   removals:  rem_keys36[first_remove .. +n_remove) and rem_entries, in window input order
 *   additions: add_keys36[first_add .. +n_add) and add_entries, in window output order
 * Every entry's script_off points into `bytes` (group after group, each group's removal scripts before its addition scripts).
 * Forward for group g is kgv_utxo_apply_diff(rem = its removal keys, add = its additions); rollback is kgv_utxo_apply_diff(rem = its addition keys,
 * add = its removal keys and entries) - on a plain table or on a view layer.
 * Output arrays (ranges included) are all host or all device memory; device entry arrays must be 8-byte aligned.  With rem_keys36 == NULL only
 * the sizes (*n_rem_out, *n_add_out, *bytes_out) and `ranges` (may be NULL) are returned; arrays smaller than that give KGV_ERR_NOMEM with the
 * sizes and ranges still set.  The three counts are host memory.  Valid under the same conditions as kgv_replay_muhash: either may come first and either may be repeated.  Without a
 * current window or with groups that do not tile it: KGV_ERR_ARG. */
typedef struct {
  uint64_t first_remove, n_remove;  /* rows of rem_keys36 / rem_entries that belong to the group */
  uint64_t first_add, n_add;        /* rows of add_keys36 / add_entries */
} kgv_diff_range; /* 32 bytes */
int kgv_replay_diffs(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, kgv_diff_range* ranges, uint8_t* rem_keys36,
                     kgv_utxo_entry* rem_entries, uint8_t* add_keys36, kgv_utxo_entry* add_entries, uint8_t* bytes, size_t max_rem, size_t max_add,
                     size_t bytes_cap, size_t* n_rem_out, size_t* n_add_out, size_t* bytes_out);
/* Overlap of the next window's upload with the current window's compute (IBD: the caller knows the blocks ahead).  A HOST batch is checked and
 * copied to the device on a side stream into a second staging buffer; the next kgv_replay_window / kgv_validate_txs / kgv_tx_ids ... call that is
 * handed exactly this batch (the same arrays and sizes) takes that buffer over instead of uploading.  The arrays must stay unchanged - and be
 * page-locked for the copy to really be asynchronous - until that call.  A device-resident batch is a no-op.  Two batches can be in flight (the
 * usual order is: prefetch window i+1, then the synchronous call for window i, whose own copy was prefetched one step earlier); a third
 * prefetch replaces the older one. */
int kgv_batch_prefetch(kgv_ctx* ctx, const kgv_tx_batch* batch);

/* ------------------------------------------------------------------------------------------------
 * Merkle roots (SURVEY.md §8f-2): crypto/merkle/src/lib.rs:3-30 calc_merkle_root / merkle_hash.
 * ------------------------------------------------------------------------------------------------ */
/* n_groups independent trees over one flattened array of 32-byte hashes: group g = hashes [first[g], first[g+1]).
 * `first` (n_groups + 1 offsets) is a HOST array; hashes32 / roots32 are both host or both device.  An empty group
 * yields ZERO_HASH, a single hash is its own root.  Serves hash_merkle_root (with kgv_tx_hashes) and
 * calc_accepted_id_merkle_root's inner root (utxo_validation.rs:401-410, with kgv_tx_ids of the accepted txs). */
int kgv_merkle_roots(kgv_ctx* ctx, const uint8_t* hashes32, const uint32_t* first, uint32_t n_groups, uint8_t* roots32);
/* calc_hash_merkle_root (consensus/core/src/merkle.rs:5-7; checked by body_validation_in_isolation.rs:34-40) for every
 * block of a batch: block b = transactions [block_first_tx[b], block_first_tx[b+1]) (host array of n_blocks + 1). */
int kgv_block_hash_merkle_roots(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks, uint8_t* roots32);

/* Block-body set checks of validate_body_in_isolation (body_validation_in_isolation.rs:13-23,95-131) for many blocks at
 * once: check_duplicate_transactions, check_block_double_spends, check_no_chained_transactions, in that order; the
 * reported item is the first offender in the reference's iteration order (the tx index for duplicates, the absolute
 * input index otherwise).  Linear work per block (the hashed sets of kgv_validate_block_bodies); any number of blocks per call. */
#define KGV_BLOCK_OK 0u
#define KGV_BLOCK_DUPLICATE_TRANSACTIONS 1u      /* RuleError::DuplicateTransactions(tx id of txs[index]) */
#define KGV_BLOCK_DOUBLE_SPEND_IN_SAME_BLOCK 2u  /* RuleError::DoubleSpendInSameBlock(inputs[index].previous_outpoint) */
#define KGV_BLOCK_CHAINED_TRANSACTION 3u         /* RuleError::ChainedTransaction(inputs[index].previous_outpoint) */
typedef struct kgv_block_check { uint32_t status, index; } kgv_block_check;
int kgv_block_set_checks(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks, kgv_block_check* out);

/* BlockBodyProcessor::validate_body_in_isolation (body_validation_in_isolation.rs:13-131) and validate_body_in_context
 * (body_validation_in_context.rs:20-80) for a window of blocks in one call.  Block b = transactions [block_first_tx[b], block_first_tx[b+1])
 * of the batch (HOST array of n_blocks + 1 offsets, monotone, from 0 to batch->n_txs), with headers[b] holding what the rules read from its
 * header and from the stores.  expected_subsidy is calc_block_subsidy(daa_score): the caller looks it up in the subsidy table it holds.
 * past_median_time is read only for a transaction whose lock time is a timestamp.  check_parent_bodies_exist is a query of the statuses
 * store and stays with the caller, before this call.
 *
 * The status of a block is its FIRST failing rule in the reference's order; a later rule is never visible when an earlier one fails:
 *   1 check_has_transactions                  NO_TRANSACTIONS
 *   2 check_hash_merkle_root                  BAD_MERKLE_ROOT          (the computed root: roots32)
 *   3 check_only_one_coinbase                 FIRST_TX_NOT_COINBASE; MULTIPLE_COINBASES with index = position in transactions[1..]
 *   4 check_transactions_in_isolation         TX_IN_ISOLATION_FAILED   index = first failing tx of the block (position in the block),
 *                                                                      tx_status = KGV_TX_* 14..30, fail_input as kgv_tx_result
 *   5 check_block_mass                        EXCEEDS_COMPUTE / TRANSIENT / STORAGE_MASS_LIMIT: index = position of the tx at which a
 *                                             running total first passes max_block_mass (at one tx compute is tested before transient
 *                                             before storage), a = that saturating total, b = max_block_mass
 *   6 check_duplicate_transactions, check_block_double_spends, check_no_chained_transactions
 *                                             DUPLICATE_TRANSACTIONS / DOUBLE_SPEND_IN_SAME_BLOCK / CHAINED_TRANSACTION, index exactly as
 *                                             kgv_block_set_checks reports it (tx resp. input index within the BATCH)
 *   7 check_coinbase_blue_score_and_subsidy   BAD_COINBASE_PAYLOAD (tx_status = KGV_COINBASE_PAYLOAD_*, a and b the CoinbaseError's two
 *                                             numbers), BAD_COINBASE_PAYLOAD_BLUE_SCORE (a payload's, b header's), WRONG_SUBSIDY
 *                                             (a expected, b payload's)
 *   8 check_block_transactions_in_context     TX_IN_CONTEXT_FAILED     index = first tx (position in the block) not finalized under ITS
 *                                                                      block's daa_score / past_median_time, tx_status =
 *                                                                      KGV_TX_NOT_FINALIZED, fail_input
 * flags: 0 runs both stages, KGV_BODY_ISOLATION_ONLY stops after rule 6 (what validate_body_in_isolation returns).
 * masses (may be NULL): the returned Mass of each block - calc_non_contextual_masses and the storage mass commitments (kgv_tx.mass), each
 * summed with saturating_add - and zeros unless the status is KGV_BODY_OK.  roots32 (may be NULL): n_blocks computed hash merkle roots
 * (bytes, any alignment).
 * rules->coinbase_payload_script_public_key_max_len also bounds the payload's script.  Every data pointer (batch, headers, results,
 * masses, roots32) host or every one device; with device pointers the call only enqueues work on the context's stream. */
typedef struct {
  uint8_t hash_merkle_root[32]; /* header.hash_merkle_root */
  uint64_t daa_score;           /* header.daa_score        */
  uint64_t blue_score;          /* header.blue_score       */
  uint64_t past_median_time;    /* calc_past_median_time_for_known_hash(block) */
  uint64_t expected_subsidy;    /* calc_block_subsidy(header.daa_score) */
} kgv_block_header_ctx; /* 64 bytes */
typedef struct {
  uint64_t max_block_mass;           /* Params::max_block_mass */
  uint64_t max_coinbase_payload_len; /* Params::max_coinbase_payload_len */
} kgv_body_rules; /* 16 bytes */
typedef struct {
  uint32_t status;     /* KGV_BODY_* */
  uint32_t index;
  uint32_t tx_status;
  uint32_t fail_input;
  uint64_t a, b;
} kgv_body_result; /* 32 bytes */
typedef struct {
  uint64_t compute_mass, transient_mass, storage_mass;
} kgv_block_masses; /* 24 bytes */
#define KGV_BODY_OK 0u
#define KGV_BODY_NO_TRANSACTIONS 1u                  /* RuleError::NoTransactions */
#define KGV_BODY_BAD_MERKLE_ROOT 2u                  /* RuleError::BadMerkleRoot(header's, computed) */
#define KGV_BODY_FIRST_TX_NOT_COINBASE 3u            /* RuleError::FirstTxNotCoinbase */
#define KGV_BODY_MULTIPLE_COINBASES 4u               /* RuleError::MultipleCoinbases(index) */
#define KGV_BODY_TX_IN_ISOLATION_FAILED 5u           /* RuleError::TxInIsolationValidationFailed(tx id, tx_status) */
#define KGV_BODY_EXCEEDS_COMPUTE_MASS_LIMIT 6u       /* RuleError::ExceedsComputeMassLimit(a, b) */
#define KGV_BODY_EXCEEDS_TRANSIENT_MASS_LIMIT 7u     /* RuleError::ExceedsTransientMassLimit(a, b) */
#define KGV_BODY_EXCEEDS_STORAGE_MASS_LIMIT 8u       /* RuleError::ExceedsStorageMassLimit(a, b) */
#define KGV_BODY_DUPLICATE_TRANSACTIONS 9u           /* RuleError::DuplicateTransactions */
#define KGV_BODY_DOUBLE_SPEND_IN_SAME_BLOCK 10u      /* RuleError::DoubleSpendInSameBlock */
#define KGV_BODY_CHAINED_TRANSACTION 11u             /* RuleError::ChainedTransaction */
#define KGV_BODY_BAD_COINBASE_PAYLOAD 12u            /* RuleError::BadCoinbasePayload(tx_status) */
#define KGV_BODY_BAD_COINBASE_PAYLOAD_BLUE_SCORE 13u /* RuleError::BadCoinbasePayloadBlueScore(a, b) */
#define KGV_BODY_WRONG_SUBSIDY 14u                   /* RuleError::WrongSubsidy(a, b) */
#define KGV_BODY_TX_IN_CONTEXT_FAILED 15u            /* RuleError::TxInContextFailed(tx id, NotFinalized(fail_input)) */
#define KGV_COINBASE_PAYLOAD_LEN_BELOW_MIN 1u        /* CoinbaseError::PayloadLenBelowMin(a = length, b = 19) */
#define KGV_COINBASE_PAYLOAD_LEN_ABOVE_MAX 2u        /* CoinbaseError::PayloadLenAboveMax(a = length, b = max_coinbase_payload_len) */
#define KGV_COINBASE_PAYLOAD_SPK_LEN_ABOVE_MAX 3u    /* CoinbaseError::PayloadScriptPublicKeyLenAboveMax(a = script length, b = maximum) */
#define KGV_COINBASE_PAYLOAD_CANT_CONTAIN_SPK 4u     /* CoinbaseError::PayloadCantContainScriptPublicKey(a = length, b = 19 + script length) */
#define KGV_BODY_ISOLATION_ONLY 1u
int kgv_validate_block_bodies(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks,
                              const kgv_block_header_ctx* headers, const kgv_tx_rules* rules, const kgv_body_rules* body_rules, uint32_t flags,
                              kgv_body_result* results, kgv_block_masses* masses, uint8_t* roots32);

/* verify_expected_utxo_state (utxo_validation.rs:182-228) for every chain block of the LAST kgv_replay_window call, with what
 * calculate_utxo_state (:110-173) gathers on the way.  Group g = blocks [group_first_block[g], group_first_block[g+1]) of that window (a HOST
 * array tiling it, as for kgv_replay_muhash) is one chain block: its first block is the selected parent (KGV_REPLAY_ACCEPT_COINBASE), then
 * the rest of the mergeset in consensus order, and its LAST block is the chain block's own body (KGV_REPLAY_VERIFY_ONLY; its transaction 0
 * is the coinbase being verified).  No other block of a group may be VERIFY_ONLY.  Any other layout (n_groups == 0 included), or no current window (see
 * kgv_replay_muhash: any other batch call or a rehash ends it) gives KGV_ERR_ARG.  The call does not end the window: it, kgv_replay_muhash
 * and kgv_replay_diffs run in any order, any number of times.
 *
 * Per group, in the reference's order, the first failing check gives results[g].status:
 *   (calculate_utxo_state, per merged block in group order)
 *     block_fee += fee overflows u64                                        REWARD_OVERFLOW
 *     its coinbase payload fails deserialize_coinbase_payload(...).unwrap()  COINBASE_PAYLOAD_UNPARSABLE
 *   1 finalize(init * multiset of groups 0..g) != headers[g].utxo_commitment BAD_UTXO_COMMITMENT
 *   2 merkle_hash(selected_parent_accepted_id_merkle_root, calc_merkle_root(accepted ids)) != accepted_id_merkle_root
 *                                                                           BAD_ACCEPTED_ID_MERKLE_ROOT
 *   4 the chain block's payload is unparsable                               COINBASE_PAYLOAD_UNPARSABLE
 *     a reward sum of expected_coinbase_transaction overflows               REWARD_OVERFLOW
 *     hashing::tx::hash(coinbase) != hash(expected_coinbase_transaction)    BAD_COINBASE_TRANSACTION
 * The REWARD_OVERFLOW and UNPARSABLE cases are the reference's panics (overflow-checks are on in its release profile; unwrap), reported at the
 * point where it panics.  Blocks that passed body validation never reach them: a payload that parses there parses here, and fees and
 * subsidies are bounded by the money supply.  Check 3 (the header's pruning point) sits between 4 and 5 in the reference and stays with the
 * caller, so check 5 is not folded into the status: n_invalid_txs / n_txs count the non-coinbase transactions of the VERIFY_ONLY block whose
 * verdict is not KGV_TX_OK, and of all of them (InvalidTransactionsInUtxoContext(n_invalid_txs, n_txs) when n_invalid_txs > 0).
 *
 * Accepted ids (ctx.accepted_tx_ids): the selected parent's coinbase, then every accepted transaction of the group's other positions, in
 * window order.  Rewards (mergeset_rewards): a merged block's subsidy is its own payload's, its total_fees the sum of the fees of its accepted
 * non-coinbase transactions.  The expected coinbase (coinbase.rs:97-142): one output of subsidy + total_fees to the block's payload script per
 * merged block that is neither red nor non-DAA, when that sum is > 0, in group order; one output of the red blocks' rewards (a non-DAA red
 * contributes its fees only) to the chain block's miner script when > 0; payload = blue_score, expected_subsidy and the chain block's own
 * miner data; version 0, no inputs, lock time 0, the coinbase subnetwork, gas 0, mass 0.
 *
 * merged_flags: one byte of KGV_MERGED_* per window block (read for the non-VERIFY_ONLY ones); the caller knows GHOSTDAG's mergeset_reds and
 * the daa_excluded store's mergeset_non_daa.  init768: (numerator || denominator) of the window's first selected parent's multiset.
 * rules->coinbase_payload_script_public_key_max_len and body_rules->max_coinbase_payload_len bound the payloads (max_block_mass is not read).
 * Outputs: results (n_groups records: the computed commitment and accepted-id root always, coinbase_hash zero when the expected coinbase could
 * not be built); block_fees (may be NULL): total_fees of every window block, 0 for VERIFY_ONLY blocks, meaningless once its sum overflowed;
 * multisets768 (may be NULL): the running (numerator || denominator) after each group - what the multiset store keeps per chain block, and
 * the next window's init768.
 * headers, merged_flags, init768, results, block_fees, multisets768: all host or all device pointers.  With device pointers the call only
 * enqueues work on the context's stream; with host pointers it synchronises once, at the end. */
typedef struct {
  uint8_t utxo_commitment[32];                         /* header.utxo_commitment */
  uint8_t accepted_id_merkle_root[32];                 /* header.accepted_id_merkle_root */
  uint8_t selected_parent_accepted_id_merkle_root[32]; /* headers_store(selected parent).accepted_id_merkle_root (utxo_validation.rs:407) */
  uint64_t blue_score;                                 /* ghostdag_data.blue_score */
  uint64_t expected_subsidy;                           /* calc_block_subsidy(header.daa_score), as in kgv_block_header_ctx */
} kgv_chain_header; /* 112 bytes */
typedef struct {
  uint32_t status;        /* KGV_CHAIN_* */
  uint32_t n_invalid_txs; /* check 5: non-coinbase transactions of the chain block that are not KGV_TX_OK */
  uint32_t n_txs;         /* non-coinbase transactions of the chain block */
  uint32_t pad_;
  uint8_t utxo_commitment[32];         /* computed */
  uint8_t accepted_id_merkle_root[32]; /* computed */
  uint8_t coinbase_hash[32];           /* hashing::tx::hash of the expected coinbase; zero if it could not be built */
} kgv_chain_result; /* 112 bytes */
#define KGV_CHAIN_OK 0u
#define KGV_CHAIN_BAD_UTXO_COMMITMENT 1u          /* RuleError::BadUTXOCommitment */
#define KGV_CHAIN_BAD_ACCEPTED_ID_MERKLE_ROOT 2u  /* RuleError::BadAcceptedIDMerkleRoot */
#define KGV_CHAIN_BAD_COINBASE_TRANSACTION 3u     /* RuleError::BadCoinbaseTransaction */
#define KGV_CHAIN_REWARD_OVERFLOW 4u              /* the reference panics: a u64 fee / reward sum overflows */
#define KGV_CHAIN_COINBASE_PAYLOAD_UNPARSABLE 5u  /* the reference panics: deserialize_coinbase_payload(...).unwrap() */
#define KGV_MERGED_RED 1u                         /* the block is in ghostdag_data.mergeset_reds */
#define KGV_MERGED_NON_DAA 2u                     /* the block is in mergeset_non_daa */
int kgv_replay_verify_chain(kgv_ctx* ctx, const uint32_t* group_first_block, size_t n_groups, const kgv_chain_header* headers, const uint8_t* merged_flags,
                            const uint8_t* init768, const kgv_tx_rules* rules, const kgv_body_rules* body_rules, kgv_chain_result* results,
                            uint64_t* block_fees, uint8_t* multisets768);

/* ------------------------------------------------------------------------------------------------
 * K8 MuHash (SURVEY.md §8f-1): crypto/muhash/src/lib.rs, u3072.rs; consensus/core/src/muhash.rs.
 * A MuHash is the pair (numerator, denominator) of residues modulo 2^3072 - 1103717 (lib.rs:32-35); every function
 * here reads / writes them as 384 little-endian bytes each, CANONICAL (in [0, p)) on output.  The reference's
 * transient non-canonical representations (u3072.rs:49-57) are unobservable through serialize()/finalize().
 * Sides of the arrays (Conventions): the two outputs of kgv_muhash_elements / kgv_muhash_txs share one; every other array of
 * these calls is on its own side, except as stated below.
 * ------------------------------------------------------------------------------------------------ */
/* MuHash::add_element / remove_element (lib.rs:61-74) for n byte strings data[offsets[i] .. offsets[i+1]):
 * remove[i] != 0 multiplies the element into the denominator, else into the numerator (remove may be NULL).
 * Starts from the empty MuHash (1, 1).  With host offsets, data and remove may each be host or device memory; with device
 * offsets (whose end, the data's size, the library cannot read) data and remove must be device memory too (KGV_ERR_ARG otherwise). */
int kgv_muhash_elements(kgv_ctx* ctx, const uint8_t* data, const uint64_t* offsets, const uint8_t* remove, size_t n, uint8_t* numerator384,
                        uint8_t* denominator384);
/* The MuHash half of validate_transactions_with_muhash_in_parallel (utxo_validation.rs:282-309): MuHash::from_transaction
 * (consensus/core/src/muhash.rs:16-27,35-39) of every tx with accept[i] != 0, all combined.  Populated entries come
 * from batch->entries, or from `table` when it is non-NULL (call BEFORE kgv_utxo_apply_accepted erases them). */
int kgv_muhash_txs(kgv_ctx* ctx, kgv_utxo_table* table, const kgv_tx_batch* batch, const uint8_t* accept, uint64_t pov_daa_score,
                   uint8_t* numerator384, uint8_t* denominator384);
/* MuHash::combine (lib.rs:91-96): a.numerator *= b.numerator, a.denominator *= b.denominator.  Each of the four arrays on its own side. */
int kgv_muhash_combine(kgv_ctx* ctx, uint8_t* numerator_a, uint8_t* denominator_a, const uint8_t* numerator_b, const uint8_t* denominator_b);
/* MuHash::serialize + finalize (lib.rs:98-115): serialized = numerator / denominator (0 has inverse 0, u3072.rs:163-165),
 * hash = BLAKE2b-256 keyed "MuHashFinalize".  Sequential by nature (one modular inversion: 3 072 dependent squarings);
 * the reference calls it once per chain block outside the parallel section.  serialized384 may be NULL.  Each array on its own side. */
int kgv_muhash_finalize(kgv_ctx* ctx, const uint8_t* numerator384, const uint8_t* denominator384, uint8_t* serialized384, uint8_t* hash32);
/* n finalizations at once: hashes32[i] = MuHash{numerator_i, denominator_i}.finalize() (lib.rs:98-115) for NONZERO denominators (every
 * denominator_i mod p != 0, which a product of hashed elements always is); value i sits pitch_bytes after value i - 1 (384 for plain
 * arrays, 768 for (numerator || denominator) records).  ONE modular inversion for the whole batch (Montgomery's trick over prefix /
 * suffix products built by parallel scans): a chain block's commitment costs five multiplications instead of 3 072 squarings.
 * serialized384 (n * 384 contiguous bytes) may be NULL.  numerators384, denominators384 and hashes32 share one side, serialized384 is on
 * its own.  KGV_ERR_ARG unless pitch_bytes >= 384 is a multiple of 16 and, for device pointers, numerators384 is 16-byte aligned and
 * hashes32 / serialized384 are 4-byte aligned. */
int kgv_muhash_finalize_batch(kgv_ctx* ctx, const uint8_t* numerators384, const uint8_t* denominators384, size_t n, size_t pitch_bytes, uint8_t* serialized384,
                              uint8_t* hashes32);
/* The MuHash::combine chain of a replay (utxo_validation.rs:144): values768 holds n (numerator || denominator) records; on return record i is
 * init * record 0 * ... * record i (canonical).  init768 may be NULL (= the empty MuHash).  A device values768 must be 16-byte aligned
 * (KGV_ERR_ARG otherwise). */
int kgv_muhash_prefix_combine(kgv_ctx* ctx, const uint8_t* init768, uint8_t* values768, size_t n);
/* MuHash::add_utxo (consensus/core/src/muhash.rs:28-33) over every live entry of the table: the UTXO-set commitment
 * numerator (denominator 1). */
int kgv_utxo_muhash(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t* numerator384);

/* ------------------------------------------------------------------------------------------------
 * Host script engine for non-standard scripts (KGV_TX_NEEDS_HOST_VM)
 * Complete restatement of TxScriptEngine (crypto/txscript/src/lib.rs:83-98,276-643, opcodes/mod.rs,
 * data_stack.rs); signature checks are resolved by a verdict provider, never computed on the CPU.
 * ------------------------------------------------------------------------------------------------ */
/* further TxScriptError variants only the full engine can produce (crypto/txscript/errors/src/lib.rs) */
#define KGV_SCRIPT_NOT_PUSH_ONLY 8
#define KGV_SCRIPT_CLEAN_STACK 9
#define KGV_SCRIPT_EMPTY_STACK 10
#define KGV_SCRIPT_ELEMENT_TOO_BIG 11
#define KGV_SCRIPT_TOO_MANY_OPERATIONS 12
#define KGV_SCRIPT_STACK_SIZE_EXCEEDED 13
#define KGV_SCRIPT_OPCODE_DISABLED 14
#define KGV_SCRIPT_OPCODE_RESERVED 15
#define KGV_SCRIPT_INVALID_OPCODE 16
#define KGV_SCRIPT_MALFORMED_PUSH 17
#define KGV_SCRIPT_MALFORMED_PUSH_SIZE 18
#define KGV_SCRIPT_NOT_MINIMAL_DATA 19
#define KGV_SCRIPT_UNBALANCED_CONDITIONAL 20
#define KGV_SCRIPT_COND_STACK_EMPTY 21    /* InvalidState("condition stack empty")       */
#define KGV_SCRIPT_EXPECTED_BOOLEAN 22    /* InvalidState("expected boolean")            */
#define KGV_SCRIPT_PICK_INVALID 23        /* InvalidState("pick at an invalid location") */
#define KGV_SCRIPT_ROLL_INVALID 24        /* InvalidState("roll at an invalid location") */
#define KGV_SCRIPT_VERIFY 25
#define KGV_SCRIPT_EARLY_RETURN 26
#define KGV_SCRIPT_INVALID_STACK_OPERATION 27
#define KGV_SCRIPT_NUMBER_TOO_BIG 28
#define KGV_SCRIPT_INVALID_PUBKEY_COUNT 29
#define KGV_SCRIPT_INVALID_SIGNATURE_COUNT 30
#define KGV_SCRIPT_UNSATISFIED_LOCKTIME 31
#define KGV_SCRIPT_SCRIPT_SIZE 32
#define KGV_SCRIPT_NO_SCRIPTS 33
#define KGV_SCRIPT_INVALID_INPUT_INDEX 34
#define KGV_SCRIPT_INVALID_OUTPUT_INDEX 35
#define KGV_SCRIPT_SERIALIZATION 36
#define KGV_SCRIPT_NEEDS_SIG_VERDICTS 254 /* kgv_script_execute only: the provider did not know a verdict */

typedef struct {
  uint32_t tx, input;      /* absolute input index into batch->inputs */
  uint8_t hash_type, ecdsa;
  uint8_t key_len;         /* 32 or 33 */
  uint8_t pad_;
  uint8_t key[33];
  uint8_t sig[64];
  uint8_t pad2_[3];
} kgv_sig_request; /* 112 bytes */
/* returns KGV_SIG_* (0..3), or a negative value if the verdict is not available */
typedef int (*kgv_verdict_fn)(void* user, const kgv_sig_request* request);

/* TxScriptEngine::from_transaction_input(..).execute() for ONE input of a HOST-resident populated batch
 * (lib.rs:276-300,399-449); `input_index` is relative to the transaction.  No GPU context is involved:
 * every check_schnorr/ecdsa_signature (lib.rs:574-643) asks `verdict` (a SigCache, the GPU batch, ...).
 * *script_err receives a KGV_SCRIPT_* code (0 = the input's scripts succeed). */
int kgv_script_execute(const kgv_tx_batch* batch, uint32_t tx, uint32_t input_index, kgv_verdict_fn verdict, void* user, uint8_t* script_err);

/* check_scripts (tx_validation_in_utxo_context.rs:162-200) with the full host engine for the listed
 * transactions of a HOST-resident populated batch; the signature checks the scripts reach are gathered,
 * hashed and verified on the GPU in batches (as many rounds as the scripts' control flow needs).
 * results[i] belongs to tx_indices[i]: status KGV_TX_OK / KGV_TX_SIGNATURE_INVALID / KGV_TX_SIGNATURE_EMPTY. */
int kgv_check_scripts_host(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* tx_indices, size_t n, kgv_tx_result* results);

/* The same check_scripts with the full script engine on the device: the same results as kgv_check_scripts_host for every input, but
 * the populated batch may be host OR device memory, and tx_indices / results may each be host or device memory.  Every input of a listed
 * transaction runs on the GPU; the signature checks its scripts reach are hashed and verified in rounds (through the attached SigCache,
 * if any), one synchronisation per round, at most 256 rounds.  This is what a caller runs after kgv_validate_populated reports
 * KGV_TX_NEEDS_HOST_VM for a device-resident batch; the table-backed calls (kgv_validate_txs, kgv_validate_mempool_txs,
 * kgv_replay_window) run the same engine internally.  An index >= batch->n_txs is refused (KGV_ERR_ARG) whichever side tx_indices is on. */
int kgv_check_scripts(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* tx_indices, size_t n, kgv_tx_result* results);

/* ------------------------------------------------------------------------------------------------
 * Persistence formats either side of the path (SURVEY.md §8f-4): the RocksDB rows of DbUtxoSetStore.  Host functions (the store lives on
 * the host): what a shim runs between the database and kgv_utxo_apply_diff / kgv_utxo_lookup (write_diff_batch utxo_set.rs:107-112, the
 * iterator feeding the pruning-point UTXO-set import processor.rs:1126-1200).
 *   key row    txid(32) || index u32 LE with trailing zero bytes trimmed, at least one kept (UtxoKey, utxo_set.rs:31-62) - WITHOUT the store's
 *              prefix bytes, which the caller prepends
 *   value row  bincode::serialize(&UtxoEntry) (database/src/access.rs:139): amount u64 || spk version u16 || script length u64 || script ||
 *              block_daa_score u64 || is_coinbase u8, all little-endian
 * Rows are packed back to back; *_off has n + 1 entries.  encode: key_rows / value_rows may be NULL (with capacity 0) to size the buffers first.
 * decode: scripts are appended to bytes_out and entries[i].script_off points there; malformed rows -> KGV_ERR_ARG.
 * ------------------------------------------------------------------------------------------------ */
int kgv_utxo_rows_encode(const uint8_t* keys36, const kgv_utxo_entry* entries, const uint8_t* bytes, size_t n_bytes, size_t n, uint8_t* key_rows, uint64_t* key_off,
                         uint8_t* value_rows, uint64_t* value_off, size_t key_cap, size_t value_cap);
int kgv_utxo_rows_decode(const uint8_t* key_rows, const uint64_t* key_off, const uint8_t* value_rows, const uint64_t* value_off, size_t n, uint8_t* keys36,
                         kgv_utxo_entry* entries, uint8_t* bytes_out, size_t bytes_cap, size_t* bytes_used);

/* ------------------------------------------------------------------------------------------------
 * Block headers in isolation: the block hash, kHeavyHash proof of work and block level of a batch of headers
 * (HeaderProcessor::validate_header_in_isolation, consensus/src/pipeline/header_processor/pre_ghostdag_validation.rs:17-24).
 * Each header is independent and needs no store.  Ordering (GHOSTDAG, DAA / difficulty, parent existence and relations) stays
 * with the caller.
 * Header k's expanded parents_by_level (ParentsByLevel::expanded_iter, consensus/core/src/header.rs:45-47) is given by
 * level_len[levels_off .. levels_off + n_levels), the number of parents at each level, and the parent hashes of all its levels
 * in order at parents32 + 32 * parents_off.  Headers may share or reorder arena ranges.  An arena range that leaves level_len
 * (n_level_entries entries) or parents32 (n_parents hashes) gives KGV_ERR_ARG whichever side the arrays are on.  The arrays of one
 * call (headers, parents32, level_len and the outputs) are all host or all device; as device memory, headers, parents32 and the
 * outputs must be 8-byte aligned and level_len 4-byte aligned (KGV_ERR_ARG otherwise).  The rules struct is host memory.  Both calls end with a synchronise of the
 * context's stream, also on device pointers: the arena ranges are checked by the kernels, and the call reports what they found.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  uint8_t hash_merkle_root[32];
  uint8_t accepted_id_merkle_root[32];
  uint8_t utxo_commitment[32];
  uint8_t pruning_point[32];
  uint8_t blue_work[24];   /* BlueWorkType (Uint192), big-endian                          */
  uint64_t timestamp;      /* milliseconds                                                */
  uint64_t nonce;
  uint64_t daa_score;
  uint64_t blue_score;
  uint64_t parents_off;    /* first parent hash of level 0, in hashes from parents32      */
  uint32_t levels_off;     /* first entry of the level sizes in level_len                */
  uint32_t n_levels;       /* expanded_len(); 0 = genesis-shaped (no parents)            */
  uint32_t bits;
  uint16_t version;
  uint16_t pad_;
} kgv_header; /* 208 bytes */

#define KGV_HEADER_SKIP_POW 1 /* kgv_header_rules.flags: skip_proof_of_work (pre_ghostdag_validation.rs:105) */
typedef struct {
  uint64_t timestamp_deviation_tolerance; /* seconds                                                              */
  uint64_t now_ms;                        /* the clock unix_now() reads in the reference, given so results repeat */
  uint32_t block_version;                 /* constants::BLOCK_VERSION                                             */
  uint32_t max_block_parents;
  uint32_t max_block_level;               /* params.max_block_level (BlockLevel, at most 255)                     */
  uint32_t flags;                         /* KGV_HEADER_*                                                         */
} kgv_header_rules; /* 32 bytes */

/* the first failing rule, in the order validate_header_in_isolation checks them; a and b carry the error's numbers */
#define KGV_HEADER_OK 0
#define KGV_HEADER_WRONG_BLOCK_VERSION 1            /* WrongBlockVersion(a = version)                              */
#define KGV_HEADER_TIME_TOO_FAR_INTO_THE_FUTURE 2   /* TimeTooFarIntoTheFuture(a = timestamp, b = max block time)  */
#define KGV_HEADER_NO_PARENTS 3                     /* NoParents                                                   */
#define KGV_HEADER_TOO_MANY_PARENTS 4               /* TooManyParents(a = level-0 parents, b = max_block_parents)  */
#define KGV_HEADER_ORIGIN_PARENT 5                  /* OriginParent                                                */
#define KGV_HEADER_INVALID_POW 6                    /* InvalidPoW                                                  */
typedef struct {
  uint32_t status;      /* KGV_HEADER_*                                                                       */
  uint8_t level;        /* calc_level_from_pow (consensus/pow/src/lib.rs:72-75); max_block_level for genesis   */
  uint8_t pow_passed;   /* pow <= target (lib.rs:47-52); 1 for genesis (lib.rs:62-64)                        */
  uint16_t pad_;
  uint64_t a, b;
} kgv_header_result; /* 24 bytes, written for every header whatever its status */

/* hashing::header::hash (consensus/core/src/hashing/header.rs:33-35) into hash32 and hash_override_nonce_time(h, 0, 0) (:7-30), the
 * pre-PoW hash, into pre_pow32; either output may be NULL.  headers, parents32, level_len and the outputs share one side; as device
 * memory, headers, parents32 and the outputs must be 8-byte aligned and level_len 4-byte aligned (KGV_ERR_ARG otherwise). */
int kgv_hash_headers(kgv_ctx* ctx, const kgv_header* headers, size_t n, const uint8_t* parents32, size_t n_parents, const uint32_t* level_len,
                     size_t n_level_entries, uint8_t* hash32, uint8_t* pre_pow32);
/* validate_header_in_isolation (pre_ghostdag_validation.rs:17-24,30-68,102-106) of every header: version, timestamp against now_ms +
 * tolerance, level-0 parent count, origin parent, then the proof of work (kaspa_pow::State::check_pow, consensus/pow/src/lib.rs:23-53:
 * pre-PoW hash, matrix from xoshiro256++ redrawn until its rank is 64, cSHAKE256 "ProofOfWorkHash", kHeavyHash, pow <= the compact
 * target).  With KGV_HEADER_SKIP_POW an insufficient proof of work is not an error; the level is still computed.  results: one record
 * per header.  hash32 (the block hash) and pow32 (the PoW value, 32 bytes little-endian) may be NULL.  Sides and alignment as for
 * kgv_hash_headers; rules is host memory. */
int kgv_validate_headers_in_isolation(kgv_ctx* ctx, const kgv_header* headers, size_t n, const uint8_t* parents32, size_t n_parents, const uint32_t* level_len,
                                      size_t n_level_entries, const kgv_header_rules* rules, kgv_header_result* results, uint8_t* hash32, uint8_t* pow32);

/* Test / audit hook: the proof-of-work matrix code on the device.  Host pointers only.
 *   op 0: Matrix::compute_rank (consensus/pow/src/matrix.rs:141-174) of n caller matrices: in = n x 64 x 64 u16 (row-major), each
 *         element converted to f64 as convert_to_float does; out = n u32 ranks.
 *   op 1: Matrix::generate (matrix.rs:103-111) from n 32-byte seeds: out = n records of 4096 u8 elements (row-major) followed by a u32
 *         count of the matrices drawn (4100 bytes each). */
int kgv_debug_pow_matrix(kgv_ctx* ctx, int op, const uint8_t* in, size_t n, uint8_t* out);

/* Test / audit hook: affine coordinates (x||y, 32-byte big-endian each) of entry v (1..65535) of
 * generator table `which` (0: v*G, 1: v*2^128*G) as built on the device. */
int kgv_gtable_entry(kgv_ctx* ctx, int which, uint32_t v, uint8_t out_xy[64]);

/* Test / audit hook: verifies ONE Schnorr triple (host pointers) on the device and returns the
 * traced intermediates: trace_words[stage*16 + i], KGV_TRACE_STAGES stages of 16 u32 words
 * (stage numbering in csrc/kgv_verify.cuh).  tests/ compare it with the host build of the same
 * device code to localise a divergence. */
#define KGV_TRACE_STAGES 32
int kgv_debug_schnorr_trace(kgv_ctx* ctx, const uint8_t* pk32, const uint8_t* msg32, const uint8_t* sig64, uint32_t* trace_words,
                            uint8_t* status);

/* Test / audit hook: which key form the last verify launch of one kind took.  A verify launch
 * decides on the device, from the number of distinct keys it counts, whether every item computes
 * its key part inline, reads a plain key record, or reads a four-tooth comb record; that choice
 * selects the scalar-multiplication ladder.  ecdsa: 0 = the last kgv_schnorr_verify launch, 1 =
 * the last kgv_ecdsa_verify launch, including launches made by the validation calls when they do
 * not go through a signature cache.  Synchronises the stream that launch ran on (which must still
 * exist) and copies one counter back: not for timed paths.  distinct_keys is the count of the
 * launch's key-deduplication pass; once it exceeds what the records allow the pass stops
 * counting, so it is then a lower bound.  KGV_ERR_ARG if no launch of that kind was made. */
#define KGV_KEY_FORM_NO_CACHE 0 /* at most one item per thread: no key deduplication ran      */
#define KGV_KEY_FORM_INLINE 1   /* deduplication ran, too many distinct keys: no records       */
#define KGV_KEY_FORM_PLAIN 2    /* one odd-multiples record per key (128-doubling ladder)     */
#define KGV_KEY_FORM_COMB 3     /* one four-tooth comb record per key (32-doubling ladder)     */
typedef struct kgv_key_form_info {
  uint64_t n_items;       /* items of the launch                                  */
  uint64_t threads;       /* threads of its grid (blocks x threads per block)     */
  uint32_t distinct_keys; /* distinct keys counted on the device (0 without cache) */
  int32_t form;           /* KGV_KEY_FORM_*                                       */
} kgv_key_form_info;
int kgv_debug_key_form(kgv_ctx* ctx, int ecdsa, kgv_key_form_info* out);
/* Signature verification rounds of the last run of the device script engine on this context (kgv_check_scripts, or the engine inside
 * kgv_validate_txs / kgv_validate_mempool_txs / kgv_replay_window); 0 when it had nothing to verify. */
int kgv_debug_script_rounds(const kgv_ctx* ctx, uint32_t* rounds);

/* Test / audit hook: runs one arithmetic primitive (its PTX body) on n operand pairs on the device.
 * in_words / out_words: n x 16 u32 (a[8] || b[8] little-endian limbs in; result limbs out).
 * op: 0 mul_wide 1 sqr_wide 2 fe_mul 3 fe_sqr 4 sc_mul 5 sc_sqr 6 sc_inv 7 fe_inv 8 fe_add 9 fe_sub
 *     10 mul_wide+reduce mod n  11 glv_split
 *     12 fe_mul_lanes 13 fe_sqr_lanes: the eight-lane forms (one item per group of eight lanes, lane k holding limb k;
 *        weakly reduced results, like 2 and 3). */
int kgv_debug_selftest(kgv_ctx* ctx, int op, const uint32_t* in_words, uint32_t* out_words, size_t n);
/* Test / audit hook: one level of the MuHash product tree on n_in caller values, by the library's own level kernel: coop = 0 the
 * one-thread-per-product multiplier, coop = 1 the 16-lane cooperative one (reduce_one otherwise picks by level size).  Host pointers
 * only; in384: n_in contiguous 384-byte little-endian values below 2^3072; out384: the (n_in + 1) / 2 raw results in[2t] * in[2t + 1]
 * folded below 2^3072 but not reduced mod p, the odd last value copied.  1 <= n_in <= 2^20. */
int kgv_debug_u3072_level(kgv_ctx* ctx, int coop, const uint8_t* in384, size_t n_in, uint8_t* out384);

#ifdef __cplusplus
}
#endif
#endif /* KGV_H */
