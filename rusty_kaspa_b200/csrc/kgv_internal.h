// kgv_internal.h — shared between the translation units of libkgv.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <condition_variable>
#include <cstdio>
#include <initializer_list>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/kgv.h"

#ifndef KGV_BLOCK
#define KGV_BLOCK 128         // threads per block of the verification kernels
#endif
#ifndef KGV_BLOCKS_PER_SM
#define KGV_BLOCKS_PER_SM 3   // 3 x 64 KiB of per-thread tables in shared memory
#endif

#ifndef KGV_ITEMS
#define KGV_ITEMS 4           // signatures per thread sharing one modular inversion (see k_schnorr_verify)
#endif

namespace kgv { struct DevEntry; }
struct ReplayRange;
struct ReplaySrc;
struct ReplayTxInfo;

struct kgv_ctx {
  int device = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t aux_stream = nullptr;              // fork/join side stream: ECDSA items verify beside the Schnorr items
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev_time[3] = {};                    // kgv_replay_window: phase timing for kgv_replay_stats
  cudaEvent_t ev_chunk[32] = {};                  // upload-complete events of the chunked host-pointer verify path
  cudaStream_t stream = nullptr;
  uint32_t* gtab = nullptr;     // [8][65536][16] u32: v*2^(32j)*G in table j, affine
  uint8_t* d_io = nullptr;      // device stand-ins of a call's host arrays (kgv_io only)
  size_t d_io_cap = 0;
  uint8_t* d_in = nullptr;      // per-call device scratch (verify uploads, signature items, script rounds, merkle trees)
  size_t d_in_cap = 0;
  uint8_t* d_out = nullptr;     // per-call device scratch (verify statuses, the script engine's phase 1)
  size_t d_out_cap = 0;
  uint8_t* d_batch = nullptr;   // staging for host-resident transaction batches
  size_t d_batch_cap = 0;
  // kgv_batch_prefetch: host batches uploaded ahead of their use on copy_stream.  Two slots, because the caller prefetches window i+1 BEFORE it
  // issues the (synchronous) call for window i, whose own prefetched copy is still waiting in the other slot.
  struct PrefetchSlot {
    uint8_t* buf = nullptr;
    size_t cap = 0;
    bool valid = false;
    const void *txs = nullptr, *inputs = nullptr, *outputs = nullptr, *entries = nullptr, *bytes = nullptr;
    size_t n_txs = 0, n_inputs = 0, n_outputs = 0, n_bytes = 0;
    cudaEvent_t done = nullptr;   // upload finished
    std::thread worker;           // range checks + upload run here, off the caller's critical path; joined by whoever consumes / reuses the slot
    int rc = 0;
    std::string err;
  } prefetch[2];
  int prefetch_next = 0;          // slot the next kgv_batch_prefetch overwrites when both are taken
  cudaEvent_t ev_prefetch = nullptr;
  cudaStream_t copy_stream = nullptr;  // its own stream: aux_stream carries the ECDSA half of a validation call
  uint8_t* d_scratch = nullptr; // per-call device scratch (sub-hashes, sig items, ...)
  size_t d_scratch_cap = 0;
  uint8_t* d_work = nullptr;    // per-call populated entries / input->tx index / verdicts of the validation calls
  size_t d_work_cap = 0;
  uint8_t* d_replay = nullptr;  // kgv_replay_window: window-wide state (tx ids, window map, script verdicts, accept mask)
  size_t d_replay_cap = 0;
  uint8_t* d_keys[2] = {};      // per-launch key cache of the verify launches (table, item slots, key records): [0] Schnorr, [1] ECDSA
  size_t d_keys_cap[2] = {};
  uint8_t* d_mu = nullptr;      // MuHash element arrays, product-tree levels and wide-product scratch rows
  size_t d_mu_cap = 0;
  // state of the last kgv_replay_window call, kept for kgv_replay_muhash / kgv_replay_diffs / kgv_replay_verify_chain (cleared by any call
  // that stages another batch)
  struct {
    bool valid = false;
    const void *txs = nullptr, *inputs = nullptr, *outputs = nullptr, *bytes = nullptr;
    size_t nt = 0, ni = 0, no = 0, n_blocks = 0;
    // the window's arrays in d_replay (kgv_replay_impl.cuh).  Read only while `valid` is set: only kgv_replay_window reserves d_replay, and
    // it clears `valid` first (kgv_batch_to_device), so these never outlive the buffer they point into.
    const uint64_t* ids = nullptr;
    const uint32_t *itx = nullptr, *otx = nullptr, *txb = nullptr;
    const uint8_t* acc = nullptr;
    const unsigned long long* apv = nullptr;
    const kgv::DevEntry* ent = nullptr;
    const ReplayRange* rng = nullptr;
    const ReplaySrc* src = nullptr;
    const ReplayTxInfo* inf = nullptr;
    const kgv_replay_block* blk = nullptr;
    const kgv_tx_result* res = nullptr;
    std::vector<uint32_t> block_flags, block_n_txs;  // host copy of the blocks' flags and sizes
    struct kgv_utxo_table* table = nullptr;          // the table replayed into, and the rehashes of its layers then: the populated entries'
    uint64_t rehashes = 0;                           // long scripts lie in those layers' arenas
  } last_replay;
  struct kgv_sigcache* sigcache = nullptr;  // kgv_set_sigcache: verdicts of the validation calls are looked up / remembered here
  struct kgv_keycache* keycache = nullptr;  // the context's attachment to a key cache (kgv_keycache_create / _share, kgv_lib.cu)
  struct kgv_comm* shard_comm = nullptr;  // kgv_set_sharding: signature checks of the validation calls are split over its ranks
  std::vector<uint8_t*> parked;  // outgrown per-call buffers, released when the caller synchronises / destroys the context (kgv_reserve)
  // tables whose arrays a write of this context gave up (rehash, growth): released from the table's list at kgv_synchronize / kgv_destroy
  std::vector<std::shared_ptr<struct kgv_table_sync>> retiring;
  uint64_t launches = 0;
  uint32_t last_script_rounds = 0;  // verification rounds of the last device script engine run (kgv_debug_script_rounds)
  // the last non-indexed verify launch of each kind ([0] Schnorr, [1] ECDSA), for kgv_debug_key_form
  struct {
    size_t n = 0;
    unsigned blocks = 0;
    bool key_cache = false;
    cudaStream_t stream = nullptr;
  } last_verify[2];
  int resident_blocks = 132 * KGV_BLOCKS_PER_SM;  // verification kernels: blocks that fit the device at once (persistent grid)
  std::recursive_mutex mu;  // recursive: an entry point may call others (kgv_check_scripts_host -> kgv_sighash, kgv_*_verify)
  std::string err;
};

int kgv_ptr_is_device(const void* p);
// KGV_ERR_ARG, with a message naming `call` and the argument `what`, when p is device memory (an argument the call reads on the host);
// KGV_OK for host memory and for null
int kgv_host_only(kgv_ctx* ctx, const char* call, const char* what, const void* p);
// cudaMalloc; under memory pressure the parked buffers are given back (after synchronising the context's streams) and the allocation retried
int kgv_malloc(kgv_ctx* ctx, void** p, size_t bytes);
int kgv_reserve(kgv_ctx* ctx, uint8_t** buf, size_t* cap, size_t need);

// returns KGV_ERR_CUDA from the enclosing function (which has `ctx` in scope) when a CUDA call fails
#define CK(call)                                                                                  \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) {                                                                      \
      char b_[256];                                                                               \
      snprintf(b_, sizeof b_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      ctx->err = b_;                                                                              \
      return KGV_ERR_CUDA;                                                                        \
    }                                                                                             \
  } while (0)

static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
static inline unsigned nblk(size_t n, unsigned b) { return (unsigned)((n + b - 1) / b); }
static inline int fail_arg(kgv_ctx* ctx, const char* m) {
  if (ctx) ctx->err = m;
  return KGV_ERR_ARG;
}

// ---- a call's device scratch, declared once ----
// A cursor over a buffer: take<T>(n, pad) hands out T[n] plus pad bytes at the cursor, and the next array starts 256-byte aligned after it.
// With a null base it only measures (every pointer is null, `at` ends at the layout's size).  A layout is one function of a kgv_carve&
// that takes its arrays in order; run once to measure and once on the buffer, it gives the size and the pointers from the same code.
struct kgv_carve {
  uint8_t* base = nullptr;  // null: measure only
  size_t at = 0;
  template <class T> T* take(size_t n, size_t pad_bytes = 0) {
    T* p = base ? (T*)(base + at) : nullptr;
    at = al256(at + n * sizeof(T) + pad_bytes);
    return p;
  }
};
// Runs lay(c) to measure, reserves *buf (kgv_reserve) to at least that size, and runs lay(c) again on the buffer.
template <class F> int kgv_reserve_carved(kgv_ctx* ctx, uint8_t** buf, size_t* cap, F&& lay) {
  kgv_carve m;
  lay(m);
  if (int rc = kgv_reserve(ctx, buf, cap, m.at)) return rc;
  kgv_carve c{*buf};
  lay(c);
  return KGV_OK;
}

// ---- where a call's caller-owned arrays live (include/kgv.h, Conventions) ----
// A call declares every array it reads (in) or writes (out) before it stages anything.  stage() gives each host array a device stand-in
// in ctx->d_io (one kgv_reserve per call) and uploads the host inputs on ctx->stream; a device array is used where it is.  copy_out()
// enqueues a copy of a device result into a caller's array of either kind.  finish() copies the host outputs back and synchronises
// ctx->stream once, only when some output (of out or copy_out) is host memory; device outputs leave the call enqueued.
//
// Which arrays of a call must share a side (one_side), which are fixed to one, and which are each on their own side (the rest).  A host-only
// argument given as device memory, or a device-only one given as host memory, is refused (KGV_ERR_ARG, naming the call and the argument)
// before it is first read.  tests/test_gpu_residency.py restates this table; its side matrix (every allowed and every forbidden
// assignment) covers the calls listed in BUILDERS there, and the host-only / device-only refusals of the others.
//   kgv_schnorr_verify, kgv_ecdsa_verify     pk, msg, sig, status together (large host batches upload in chunks on the side stream)
//   kgv_status_to_bitmap                     status, bitmap together
//   kgv_tx_ids, kgv_tx_hashes                out32 on its own side
//   kgv_sighash                              items and out32 together, independent of the batch
//   kgv_merkle_roots                         hashes32 and roots32 together; first on the host
//   kgv_block_hash_merkle_roots,
//   kgv_block_set_checks                     the output on its own side; block_first_tx on the host
//   kgv_muhash_elements                      numerator384 and denominator384 together; with host offsets data and remove each on their own
//                                            side, with device offsets data and remove on the device too
//   kgv_muhash_combine, kgv_muhash_finalize  every input and every output on its own side
//   kgv_muhash_finalize_batch                numerators384, denominators384, hashes32 together, serialized384 on its own side; device
//                                            numerators384 16-byte aligned, device hashes32 and serialized384 4-byte aligned
//   kgv_muhash_prefix_combine                values768 (updated in place, 16-byte aligned on the device) and init768 each on their own side
//   kgv_muhash_txs                           numerator384 and denominator384 together; accept on its own side
//   kgv_utxo_muhash                          numerator384 on its own side
//   kgv_utxo_lookup / _apply_diff            each array on its own side
//   kgv_utxo_export                          each array on its own side; n_out and bytes_out on the host
//   kgv_utxo_count, kgv_utxo_digest,
//   kgv_utxo_stats, kgv_sigcache_counters    the results on the host
//   kgv_utxo_import_chunk                    numerator384 on the host; keys36, entries, bytes each on their own side (the script ranges of
//                                            entries are checked on either side)
//   kgv_utxo_apply_accepted                  accept on its own side (a host accept: the call waits for the table)
//   kgv_validate_txs, kgv_validate_populated results on its own side, independent of the batch; params on the host
//   kgv_validate_mempool_txs*                results, batch->txs, args, storage_mass, entries_out, scripts_out, masses, detail together;
//                                            params, rules, policy and scripts_used on the host
//   kgv_validate_txs_in_isolation            results, batch->txs, masses together; rules on the host
//   kgv_check_txs_standard_in_isolation      results, batch->txs, masses, detail together; the policy on the host
//   kgv_check_txs_standard_in_context        results, batch->txs, masses, storage_mass, fee, detail together; the policy on the host
//   kgv_outputs_dust                         is_dust and batch->outputs together
//   kgv_validate_block_bodies                results, batch->txs, headers, masses, roots32 together; block_first_tx, rules and body_rules on
//                                            the host
//   kgv_hash_headers, kgv_validate_headers_in_isolation
//                                            headers, parents32, level_len and the outputs together, device arrays 8-byte aligned (level_len
//                                            4-byte); rules on the host
//   kgv_replay_window                        blocks, params and stats on the host; results and accept each on their own side
//   kgv_replay_muhash                        values768 on its own side; group_first_block on the host
//   kgv_replay_diffs                         the output arrays together (ranges alone when counting), device entry arrays 8-byte aligned;
//                                            group_first_block and the counts on the host
//   kgv_replay_verify_chain                  results, headers, merged_flags, init768, block_fees, multisets768 together (inputs are copied into
//                                            the call's own workspace from either side); group_first_block, rules and body_rules on the host
//   kgv_check_scripts                        tx_indices and results each on their own side (the indices are range-checked on either side)
//   the kgv_comm.cu calls                    device arrays only; epoch_out on the host
// The arrays of a transaction batch are staged by kgv_batch_to_device (d_batch, or a prefetch slot) and must all be of one kind.
class kgv_io {
 public:
  explicit kgv_io(kgv_ctx* c) : ctx(c) {}
  // KGV_ERR_ARG, with a message naming `call`, unless the non-null pointers are all host or all device memory; *dev (may be null): their side
  int one_side(const char* call, std::initializer_list<const void*> ps, bool* dev = nullptr);
  bool is_device(const void* p);  // queried once per pointer and call
  // *d = the array's device address: p itself for device memory (or null p), its stand-in after stage() for host memory
  template <class T> void in(const T* p, size_t bytes, const T** d) { add(p, bytes, (const void**)d, true, false); }
  template <class T> void out(T* p, size_t bytes, T** d) { add(p, bytes, (const void**)d, false, true); }
  template <class T> void inout(T* p, size_t bytes, T** d) { add(p, bytes, (const void**)d, true, true); }  // updated in place
  int stage();
  int copy_out(void* p, const void* d, size_t bytes);
  void trim(const void* p, size_t bytes);  // a declared output comes back only up to `bytes` (sizes known after the kernels)
  int finish();

 private:
  void add(const void* p, size_t bytes, const void** d, bool in, bool out);
  kgv_ctx* ctx;
  struct Arr { const void* p; size_t bytes; const void** d; bool in, out; };
  Arr arr[10];          // the host arrays of the call
  int n_arr = 0;
  struct Side { const void* p; bool dev; } side[16];
  int n_side = 0;
  bool host_out = false;
};

// ---- transaction batches on the device (kgv_hash.cu) ----
struct kgv_dev_batch {
  const kgv_tx* txs;
  const kgv_input* inputs;
  const kgv_output* outputs;
  const kgv_utxo_entry* entries;
  const uint8_t* bytes;
  size_t n_txs, n_inputs, n_outputs, n_bytes;
};
// Makes the batch arrays device-resident (uploads host arrays into ctx staging; wraps device arrays).
int kgv_batch_to_device(kgv_ctx* ctx, const kgv_tx_batch* b, kgv_dev_batch* out, bool need_entries);

// Enqueue a verification kernel on device-resident SoA item arrays on stream st (no locking, no copies): used by the
// fused validation path.  ecdsa: pk stride 33, else 32.
int kgv_launch_verify(kgv_ctx* ctx, const uint8_t* dpk, const uint8_t* dmsg, const uint8_t* dsig, size_t n, uint8_t* dstatus, bool ecdsa,
                      cudaStream_t st, const uint32_t* index = nullptr, const uint32_t* n_dev = nullptr);

// ---- MuHash product trees (kgv_muhash.cu) ----
// Reserve the level-0 element arrays of the two trees (denominator = removed elements, numerator = added elements):
// element e of a tree with n elements has its limb block i at E + (i*n + e)*8 words (kgv_u3072.cuh layout, stride n).
int kgv_mu_reserve(kgv_ctx* ctx, size_t n_den, size_t n_num, uint32_t** e_den, uint32_t** e_num);
// Multiply each tree down to one value (denominator on ctx->stream, numerator on the side stream) and write the two
// canonical residues (384 little-endian bytes each) to host or device memory.
int kgv_mu_reduce(kgv_ctx* ctx, kgv_io& io, size_t n_den, size_t n_num, uint8_t* out_num384, uint8_t* out_den384);
// out + g * out_pitch_words = product of the level-0 elements E[lo[g] .. hi[g]) with flags[flag_index[j]] != 0 (one 16-lane group per range)
int kgv_mu_range_products(kgv_ctx* ctx, const uint32_t* E, size_t stride, const uint8_t* flags, const uint32_t* flag_index, const uint32_t* lo, const uint32_t* hi, uint32_t n_segs,
                          uint32_t* out, size_t out_pitch_words, cudaStream_t st);
int kgv_mu_canonicalize(kgv_ctx* ctx, uint32_t* vals, size_t pitch_words, size_t n, cudaStream_t st);
// kgv_muhash_prefix_combine on device records (v: n (numerator || denominator) records, 16-byte aligned; dinit: one record or null), in place
struct kgv_mu_prefix_work { uint32_t* tot; void carve(kgv_carve& c, size_t n); };  // tot: the scan's chunk totals
int kgv_mu_prefix_combine_run(kgv_ctx* ctx, const uint32_t* dinit, uint32_t* v, size_t n, const kgv_mu_prefix_work& w, cudaStream_t st);
// kgv_muhash_finalize_batch on device values (numerator k at dnum + k * pitch_words, 16-byte aligned); dser (may be null) / dhashes: n values
// of 384 / 32 bytes, 4-byte aligned
struct kgv_mu_finalize_work {  // prefix and suffix products, the quotients, the scan's chunk totals, the inversion's operands
  uint32_t *P, *S, *out, *tot, *inv;
  void carve(kgv_carve& c, size_t n);
};
int kgv_mu_finalize_run(kgv_ctx* ctx, const uint32_t* dnum, const uint32_t* dden, size_t n, size_t pitch_words, const kgv_mu_finalize_work& w,
                        uint32_t* dser, uint32_t* dhashes, cudaStream_t st);
// kgv_replay_muhash on the last window's state (kgv_validate.cu): dgf = n_groups + 1 device block offsets; vals = n_groups canonical
// (numerator || denominator) records, 768 bytes apart, 16-byte aligned.  The element arrays live in d_mu.
struct kgv_replay_muhash_work {  // per transaction its block's DAA score and whether it is the block's first; per group its input / output range
  uint64_t* pov;
  uint8_t* first;
  uint32_t *ilo, *ihi, *olo, *ohi;
  void carve(kgv_carve& c, size_t nt, size_t n_groups);
};
int kgv_replay_muhash_run(kgv_ctx* ctx, const uint32_t* dgf, size_t n_groups, const kgv_replay_muhash_work& w, uint32_t* vals, cudaStream_t st);

// ---- one UTXO table used from every context of its device (kgv_utxo_maint.cu; include/kgv.h, "Threading") ----
// A reader/writer lock per table whose ordering lives on the GPU.  A call registers before it enqueues the first work that touches the
// table and drops the registration after the last.  A read makes its stream wait for the event that ends the last write; the host does
// not block unless a write is open or queued.  A write waits on the host until the reads of OTHER contexts have dropped (the reference's
// upgrade()), makes its stream wait for their events and the last write's, and records the new last-write event when it drops.  Writers
// enter in ticket order and readers wait while one is queued, so a steady stream of reads cannot starve a commit.  Registration is
// reentrant per context (entry points call each other under the context's recursive mutex); a read inside the context's own write is part
// of that write.
struct kgv_table_sync {
  int device = 0;
  std::mutex m;
  std::condition_variable cv;
  struct Reader { const kgv_ctx* ctx; int depth; };
  std::vector<Reader> readers;            // open read registrations
  const void* writer = nullptr;           // the context whose write is open (write_depth > 0)
  int write_depth = 0;
  uint64_t next_ticket = 0, serving = 0;  // writers queued or open: next_ticket - serving
  cudaEvent_t last_write = nullptr;       // ends the last write
  std::vector<std::pair<cudaStream_t, cudaEvent_t>> reads;  // end the reads since that write: one event per stream, re-recorded
  std::vector<cudaEvent_t> pool;          // cudaEventDisableTiming events not in use
  uint64_t writes = 0;
  std::vector<void*> retiring;            // arrays the open write gave up
  cudaEvent_t retire_ev = nullptr;        // (reserved for them by kgv_table_retire)
  struct Retired { cudaEvent_t done; std::vector<void*> ptrs; };
  std::vector<Retired> retired;           // freed once `done` has completed
  ~kgv_table_sync();                      // destroys the events left (the lock's users have finished on the GPU)
};
struct kgv_utxo_table;
// The registrations of one call, dropped (events recorded on the stream each was taken for: ctx->stream for tables) when it goes out of scope.
class kgv_table_access {
 public:
  explicit kgv_table_access(kgv_ctx* c) : ctx(c) {}
  ~kgv_table_access() { release(); }
  kgv_table_access(const kgv_table_access&) = delete;
  kgv_table_access& operator=(const kgv_table_access&) = delete;
  // A read on every layer of t's view chain, except `written` (a layer of it, or null) which gets a write; bottom layer first, so calls
  // that touch several tables cannot deadlock.  KGV_ERR_ARG, naming `call`, when a layer belongs to another device than the context.
  int acquire(const char* call, kgv_utxo_table* t, kgv_utxo_table* written = nullptr);
  // A read (or a write) of one bare lock for work enqueued on st, whose release event is recorded there (the key cache's partitions).
  int acquire(kgv_table_sync* s, bool write, cudaStream_t st);
  void release();

 private:
  enum Mode { kNone, kRead, kWrite };
  int lock(kgv_table_sync* s, Mode m, cudaStream_t st);
  kgv_ctx* ctx;
  struct Held { kgv_table_sync* s; Mode m; cudaEvent_t ev; cudaStream_t st; };
  std::vector<Held> held;
};
// Hands an array of t to the table's release list: freed after the open write of ctx (which gave it up) has completed on the GPU.
int kgv_table_retire(kgv_ctx* ctx, kgv_utxo_table* t, void* p);
// kgv_replay_muhash / _diffs / _verify_chain: a read of the layers of the last replay window's table, refused (KGV_ERR_ARG, naming `call`) when
// one of them was rehashed since by any context.
int kgv_last_replay_read(kgv_ctx* ctx, kgv_table_access& acc, const char* call);
uint64_t kgv_chain_rehashes(const kgv_utxo_table* t);
// Frees the retired arrays of the tables this context wrote whose writes have completed; wait: wait for the others and free them too.
void kgv_release_retired(kgv_ctx* ctx, bool wait);

// ---- shared pieces of the validation path (kgv_validate.cu) ----
// Growth policy of a table (kgv_utxo_set_max_load, kgv_utxo_maint.cu): called by every table writer before it writes.  m bounds the slots the
// call can newly occupy, b the long-script bytes it can append.  Returns at once when the policy is off; otherwise it may rehash the table
// (KGV_ERR_NOMEM when that fails: the caller returns before writing anything).
int utxo_reserve(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t m, uint64_t b);
// exclusive prefix sums of one (in1 == null) or two u32 arrays of n elements on st; totals[0] (and totals[1]) get the sums
int kgv_scan_u32(kgv_ctx* ctx, const uint32_t* in0, uint32_t* out0, const uint32_t* in1, uint32_t* out1, size_t n, uint32_t* totals, cudaStream_t st);
// the verification step of the script phase for n device-resident items (pk stride 33 for ECDSA, else 32; 32-byte messages, 64-byte
// signatures -> KGV_SIG_* in st).  With a SigCache (sc) hits are answered from it and the misses verified and inserted; dig (32 B per item),
// idx (4 B per item) and nm (one u32) are its scratch.
int kgv_verify_items(kgv_ctx* ctx, struct kgv_sigcache* sc, const uint8_t* pk, const uint8_t* msg, const uint8_t* sig, size_t n, bool ecdsa, uint8_t* st,
                     uint8_t* dig, uint32_t* idx, uint32_t* nm, cudaStream_t s);
// check_scripts with the device script engine (kgv_scripts_dev.cu) for n_list transactions of a populated device batch view: dlist holds
// their indices, or is null to take the transactions whose dres status is KGV_TX_NEEDS_HOST_VM.  patch: dres[tx] gets status / script_err /
// fail_input (the fee stays); else dres[j] = the result of list entry j.  *rounds_out (may be null): verification rounds run.
namespace kgv { struct BatchView; }
int kgv_script_engine_run(kgv_ctx* ctx, const kgv::BatchView& v, size_t n_txs, const uint32_t* dlist, size_t n_list, kgv_tx_result* dres, bool patch,
                          uint32_t* rounds_out);

// ---- isolation rules, finality and non-contextual masses (kgv_isolation.cu) ----
// Enqueues on st, for every tx of a device batch: dres = the first failing isolation / finality rule (finality == false skips it),
// dmasses = calc_non_contextual_masses and dnc = max(compute, transient) (either may be null).  dlist: scratch of n_txs + 1 u32.
// With dheaders (device, one record per block) and dtx_block (device, the block of every tx) the finality rule reads each transaction's
// own block's daa_score / past_median_time instead of daa / pmt.
int kgv_isolation_run(kgv_ctx* ctx, const kgv_dev_batch& d, const kgv_tx_rules& rules, uint64_t daa, uint64_t pmt, bool finality, kgv_tx_result* dres,
                      kgv_tx_masses* dmasses, uint64_t* dnc, uint32_t* dlist, cudaStream_t st, const kgv_block_header_ctx* dheaders = nullptr,
                      const uint32_t* dtx_block = nullptr);

// ---- the mempool's standardness policy (kgv_standard.cu) ----
// check_transaction_standard_in_isolation of every tx of a device batch on st: dres gets the verdict (with gate, only a failure is
// written), ddetail (may be null) the number it carries for every tx.  dmasses: the non-contextual masses.
int kgv_standard_isolation_run(kgv_ctx* ctx, const kgv_dev_batch& d, const kgv_mempool_policy& p, const kgv_tx_masses* dmasses, bool gate,
                               kgv_tx_result* dres, uint64_t* ddetail, cudaStream_t st);
// check_transaction_standard_in_context on st.  dent: the populated entries of a validation call, or null to read d.entries.  dfee: the
// fees, or null to check only the txs whose dres status is KGV_TX_OK with their dres fee (then only failures are written).  *dflag |= 1
// when a reached fee check's mass * fee overflows u64.
int kgv_standard_context_run(kgv_ctx* ctx, const kgv_dev_batch& d, const kgv::DevEntry* dent, const kgv_mempool_policy& p, const kgv_tx_masses* dmasses,
                             const uint64_t* dsmass, const uint64_t* dfee, kgv_tx_result* dres, uint64_t* ddetail, unsigned long long* dflag,
                             cudaStream_t st);

// ---- pieces of the block body path shared between kgv_hash.cu and kgv_block_body.cu ----
// enqueue Transaction::id() (hash == false) or hashing::tx::hash (true) of the first n txs of a device batch into out (32 B each)
int kgv_tx_digests_run(kgv_ctx* ctx, const kgv_dev_batch& d, size_t n, uint64_t* out, bool hash);
// merkle roots of n_groups groups over the device hashes dh (overwritten); first_host: n_groups + 1 offsets on the host.  Uses d_scratch.
int kgv_merkle_run(kgv_ctx* ctx, uint64_t* dh, size_t n_total, const uint32_t* first_host, uint32_t n_groups, uint64_t* droots);
// the same with DEVICE offsets dfirst (n_groups + 1, from 0 to at most n_cap hashes) and max_n >= the largest group.  Enqueued on st.
struct kgv_merkle_work { uint32_t* gid; uint64_t* other; void carve(kgv_carve& c, size_t n_cap); };  // every hash's group, the levels' second buffer
int kgv_merkle_levels(kgv_ctx* ctx, uint64_t* dh, size_t n_cap, const uint32_t* dfirst, uint32_t n_groups, uint32_t max_n, const kgv_merkle_work& w,
                      uint64_t* droots, cudaStream_t st);
// check_duplicate_transactions / check_block_double_spends / check_no_chained_transactions of every block (kgv_block_body.cu): dacc[b] gets
// the lowest offending tx / input / input index within the batch, 0xFFFFFFFF where a check passes.  dids: the tx ids; dfirst: the block
// offsets on the device.
struct kgv_block_check_acc { unsigned int dup_tx, double_spend, chained; };
struct kgv_body_sets_work {  // the blocks' hashed sets, cleared whole (up to the next 256-byte boundary)
  uint32_t* tab;
  size_t bytes;
  void carve(kgv_carve& c, size_t n_txs, size_t n_inputs);
};
int kgv_body_sets_run(kgv_ctx* ctx, const kgv_dev_batch& d, size_t n_txs, const uint64_t* dids, const uint32_t* dfirst, uint32_t n_blocks,
                      kgv_block_check_acc* dacc, const kgv_body_sets_work& w, cudaStream_t st);

// ---- multi-GPU exchange used by the sharded script phase (kgv_comm.cu) ----
// Every rank contributes `per` bytes at buf + rank * per (device memory, n_ranks * per bytes in all); on return (stream order)
// buf holds all ranks' contributions.  Peer transport if the communicator is connected, else NCCL (in place).
int kgv_comm_exchange_slices(kgv_ctx* ctx, struct kgv_comm* c, uint8_t* buf, size_t per);
int kgv_comm_ranks(const struct kgv_comm* c, int* rank);

// ---- signature cache (kgv_sigcache.cu): device verdict table keyed by BLAKE2b-256(kind || sig || pk || msg) ----
// Looks every item up; status[i] = cached verdict or 0xFF; writes the digests (32 B per item, reused by the insert), the compacted list of
// misses and their count (device).  Enqueued on `st`.
int kgv_sigcache_lookup(kgv_ctx* ctx, struct kgv_sigcache* c, const uint8_t* pk, const uint8_t* msg, const uint8_t* sig, size_t n, bool ecdsa, uint8_t* status, uint8_t* digests,
                        uint32_t* miss_index, uint32_t* n_miss_dev, cudaStream_t st);
// remembers the verdicts (0 / 1 only, as the reference: parse errors never reach its cache) of the listed items
int kgv_sigcache_insert(kgv_ctx* ctx, struct kgv_sigcache* c, const uint8_t* status, const uint8_t* digests, const uint32_t* miss_index, const uint32_t* n_miss_dev, size_t n_max,
                        cudaStream_t st);
