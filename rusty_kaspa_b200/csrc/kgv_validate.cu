// kgv_validate.cu — GPU-resident UTXO table, per-transaction context rules and the fused
// validate_transactions path (include/kgv.h).
//
// Data flow of kgv_validate_txs (one call = one block's worth or more of transactions):
//   k_populate        per input : outpoint -> table slot -> DevEntry            (HBM latency bound)
//   k_tx_context      per tx    : maturity, amounts, storage mass, seq-lock      (tx_validation_in_utxo_context.rs:75-155)
//   k_plan            per input : recognise P2PK / P2PK-ECDSA / P2SH multisig, count signature checks
//   (scan)                        exclusive prefix sums -> item offsets (two lists: Schnorr, ECDSA)
//   k_emit_items      per input : gather (pk, sig) of every candidate pair into SoA arrays
//   k_sighash_reused  per tx    : the five reusable sub-hashes                   (sighash.rs:14-221)
//   k_item_msgs       per item  : final signature hash                           (sighash.rs:238-277)
//   k_schnorr_verify / k_ecdsa_verify per item                                   (lib.rs:593, :628)
//   k_resolve         per input : replay of the script engine over the verdicts  (lib.rs:488-571)
//   k_tx_finalize     per tx    : first failing input -> TxRuleError class       (:162-200)
#include "kgv_internal.h"
#include "kgv_muhash.cuh"
#include "kgv_txhash.cuh"
#include "kgv_utxo.cuh"
#include "kgv_context.cuh"
#include "kgv_standard.cuh"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

using namespace kgv;


// KGV_DEBUG=1: synchronise and report after every stage of the fused path (locates a faulting kernel)
#include <cstdlib>
static bool kgv_debug_on() { static int v = -1; if (v < 0) v = getenv("KGV_DEBUG") ? 1 : 0; return v == 1; }
#define STAGE(name)                                                                               \
  do {                                                                                            \
    if (kgv_debug_on()) {                                                                         \
      cudaError_t e_ = cudaStreamSynchronize(ctx->stream);                                        \
      fprintf(stderr, "[kgv] stage %s: %s\n", name, cudaGetErrorString(e_));                      \
      fflush(stderr);                                                                             \
    }                                                                                             \
  } while (0)

// ---------------------------------------------------------------------------------------------
// UTXO table kernels (device functions: kgv_utxo.cuh)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void slot_to_entry(DevEntry& e, const TableView& t, const UtxoSlot* s) {
  SlotHead h;
  slot_load_head(h, s);
  head_to_entry(e, t, s, h);
}

__global__ void k_utxo_lookup(TableView t, const uint8_t* __restrict__ keys, size_t n, kgv_utxo_entry* __restrict__ entries,
                              uint8_t* __restrict__ scripts, uint32_t stride, uint8_t* __restrict__ found) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k[9];
  load_key(k, keys + 36 * i);
  SlotHead h;
  UtxoSlot* s = table_find(t, k, h);
  // the 32-byte entry record is written with two 128-bit stores
  uint32_t e[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  e[4] = (uint32_t)(i * stride);  // script_off
  if (s) {
    DevEntry d;
    head_to_entry(d, t, s, h);
    e[0] = h.w[10]; e[1] = h.w[11]; e[2] = h.w[12]; e[3] = h.w[13];
    e[5] = d.script_len;
    e[6] = (uint32_t)d.spk_version | ((uint32_t)d.is_coinbase << 16);
    for (uint32_t b = 0; b < d.script_len && b < stride; b++) scripts[i * stride + b] = d.script[b];
  }
  if ((((uintptr_t)entries) & 31) == 0) st256(entries + i, e);
  else {
    uint32_t* o = (uint32_t*)(entries + i);
#pragma unroll
    for (int j = 0; j < 8; j++) o[j] = e[j];
  }
  found[i] = s ? 1 : 0;
}
__global__ void k_utxo_erase(TableView t, const uint8_t* __restrict__ keys, size_t n, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k[9];
  load_key(k, keys + 36 * i);
  uint32_t r = table_erase(t, k);
  if (status) status[i] = (uint8_t)r;
}
__global__ void k_utxo_insert(TableView t, const uint8_t* __restrict__ keys, const kgv_utxo_entry* __restrict__ entries, const uint8_t* __restrict__ bytes,
                              size_t n, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k[9];
  load_key(k, keys + 36 * i);
  kgv_utxo_entry e = entries[i];
  uint32_t r = table_put(t, k, e.amount, e.block_daa_score, e.spk_version, e.is_coinbase, bytes + e.script_off, e.script_len);
  if (status) status[i] = (uint8_t)r;
}

// export (DbUtxoSetStore::iterator, utxo_set.rs:114-129: the syncer side of a pruning-point import and the source of `virtual.utxo_set := pruning
// utxo_set`, processor.rs:1150-1158): every live slot is compacted into (key, entry, script bytes) arrays; order is the table's, i.e. arbitrary
__global__ void k_utxo_export(TableView t, uint8_t* __restrict__ keys, kgv_utxo_entry* __restrict__ entries, uint8_t* __restrict__ bytes, uint64_t max_n, uint64_t bytes_cap,
                              unsigned long long* __restrict__ cnt) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > t.mask) return;
  const UtxoSlot* s = &t.slots[i];
  if (s->state != SLOT_FULL) return;
  DevEntry e;
  slot_to_entry(e, t, s);
  const unsigned long long at = atomicAdd(&cnt[0], 1ull);
  const unsigned long long off = atomicAdd(&cnt[1], (unsigned long long)e.script_len);
  if (!keys || at >= max_n || off + e.script_len > bytes_cap || off + e.script_len > 0xFFFFFFFFull) return;  // counting pass / caller's arrays too small (reported by the host side)
  uint32_t* kw = (uint32_t*)(keys + 36 * at);
#pragma unroll
  for (int w = 0; w < 9; w++) kw[w] = s->key[w];
  kgv_utxo_entry o;
  o.amount = e.amount; o.block_daa_score = e.block_daa_score; o.script_off = (uint32_t)off; o.script_len = e.script_len; o.spk_version = e.spk_version; o.is_coinbase = e.is_coinbase;
  memset(o.pad_, 0, sizeof o.pad_);
  entries[at] = o;
  for (uint32_t b = 0; b < e.script_len; b++) bytes[off + b] = e.script[b];
}
// MuHash::from_utxo of every (outpoint, entry) of a chunk (consensus/src/consensus/mod.rs:1075-1080): level 0 of a product tree
__global__ void __launch_bounds__(128) k_muhash_utxo_elements(const uint8_t* __restrict__ keys, const kgv_utxo_entry* __restrict__ entries, const uint8_t* __restrict__ bytes, size_t n,
                                                              uint32_t* __restrict__ e_num) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  uint32_t k[9];
  load_key(k, keys + 36 * g);
  const kgv_utxo_entry e = entries[g];
  uint64_t d[4];
  muhash_utxo_digest(d, k, k[8], e.block_daa_score, e.amount, e.is_coinbase != 0, e.spk_version, bytes + e.script_off, e.script_len);
  muhash_expand_store(e_num, n, g, d);
}

// digest: sum of MuHashElement hashes, accumulated as 8 x 32-bit limbs in 64-bit counters (carries folded on the host)
__global__ void k_utxo_digest(TableView t, unsigned long long* __restrict__ acc) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > t.mask) return;
  const UtxoSlot* s = &t.slots[i];
  if (s->state != SLOT_FULL) return;
  DevEntry e;
  slot_to_entry(e, t, s);
  Blake2b h;
  b2b_init_muhash_element(h);
  for (int w = 0; w < 9; w++) b2b_u32(h, s->key[w]);
  b2b_u64(h, e.block_daa_score);
  b2b_u64(h, e.amount);
  b2b_u8(h, e.is_coinbase ? 1 : 0);
  b2b_u16(h, e.spk_version);
  b2b_u64(h, e.script_len);
  b2b_bytes(h, e.script, e.script_len);
  uint64_t d[4];
  b2b_final(h, d);
#pragma unroll
  for (int w = 0; w < 4; w++) {
    atomicAdd(&acc[2 * w], (unsigned long long)(uint32_t)d[w]);
    atomicAdd(&acc[2 * w + 1], (unsigned long long)(uint32_t)(d[w] >> 32));
  }
}

// ---------------------------------------------------------------------------------------------
// validation kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_entries_from_batch(const kgv_utxo_entry* __restrict__ in, const uint8_t* __restrict__ bytes, size_t n, DevEntry* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  kgv_utxo_entry e = in[i];
  DevEntry d;
  d.amount = e.amount; d.block_daa_score = e.block_daa_score; d.script = bytes + e.script_off; d.script_len = e.script_len;
  d.spk_version = e.spk_version; d.is_coinbase = e.is_coinbase; d.found = e.pad_[0] ? 0 : 1;  // pad_[0] != 0: caller marks the entry absent
  out[i] = d;
}

__global__ void k_populate(TableView t, const kgv_input* __restrict__ inputs, size_t n, DevEntry* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k[9];
  input_key(k, inputs[i]);
  SlotHead h;
  UtxoSlot* s = table_find(t, k, h);
  DevEntry d;
  if (s) head_to_entry(d, t, s, h);
  else entry_absent(d);
  out[i] = d;
}

__global__ void k_tx_context(BatchView b, uint32_t n_txs, uint64_t pov, uint32_t flags, kgv_params prm, kgv_tx_result* __restrict__ res) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  res[ti] = tx_context_rules(b, ti, pov, flags, prm, tx_is_coinbase(b.txs[ti]));
}

// populate_mempool_transaction_in_utxo_context (utxo_validation.rs:341-363): an entry the caller supplies (given[i].pad_[0] == 0; its script in
// the batch arena) is kept, every other input is looked up.  len[i] = script bytes of the final entry (0 when absent); *total = their sum in
// 64 bits (the 32-bit offsets of the scan are only used when it fits).  Launched with whole warps: every lane reaches the reduction.
// gate (may be null): the isolation verdicts; an input of a transaction that failed them is never looked up (absent unless supplied).
__global__ void k_populate_mempool(TableView t, const kgv_input* __restrict__ inputs, const kgv_utxo_entry* __restrict__ given, const uint8_t* __restrict__ bytes,
                                   size_t n, DevEntry* __restrict__ out, uint32_t* __restrict__ len, unsigned long long* __restrict__ total,
                                   const kgv_tx_result* __restrict__ gate, const uint32_t* __restrict__ input_tx) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long l = 0;
  if (i < n) {
    DevEntry d;
    if (given && !given[i].pad_[0]) {
      const kgv_utxo_entry e = given[i];
      d.amount = e.amount; d.block_daa_score = e.block_daa_score; d.script = bytes + e.script_off; d.script_len = e.script_len;
      d.spk_version = e.spk_version; d.is_coinbase = e.is_coinbase; d.found = 1;
    } else if (gate && gate[input_tx[i]].status != KGV_TX_OK) {
      entry_absent(d);
    } else {
      uint32_t k[9];
      input_key(k, inputs[i]);
      SlotHead h;
      UtxoSlot* s = table_find(t, k, h);
      if (s) head_to_entry(d, t, s, h);
      else entry_absent(d);
    }
    out[i] = d;
    l = d.found ? d.script_len : 0;
    len[i] = (uint32_t)l;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) l += __shfl_down_sync(0xFFFFFFFFu, l, o);
  if ((threadIdx.x & 31) == 0 && l) atomicAdd(total, l);
}

// the context rules of a mempool batch (mempool_context_rules); *bad counts thresholds with a zero divisor.  gate (may be null): a
// transaction that failed isolation or finality keeps that verdict and a storage mass of 0; nc_mass (may be null) replaces the
// caller's args[ti].non_contextual_mass.
__global__ void k_tx_mempool_context(BatchView b, uint32_t n_txs, uint64_t pov, kgv_params prm, const kgv_mempool_tx_args* __restrict__ args,
                                     kgv_tx_result* __restrict__ res, uint64_t* __restrict__ mass, unsigned long long* __restrict__ bad,
                                     const kgv_tx_result* __restrict__ gate, const uint64_t* __restrict__ nc_mass) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  if (gate && gate[ti].status != KGV_TX_OK) { res[ti] = gate[ti]; mass[ti] = 0; return; }
  double thr = __longlong_as_double(0x7FF8000000000000ll);  // NaN: no threshold
  uint64_t nc = 0;
  if (args) { thr = args[ti].feerate_threshold; nc = args[ti].non_contextual_mass; }
  if (nc_mass) nc = nc_mass[ti];
  uint64_t m;
  bool bad_thr;
  res[ti] = mempool_context_rules(b, ti, pov, prm, thr, nc, m, bad_thr);
  mass[ti] = m;
  if (bad_thr) atomicAdd(bad, 1ull);
}

// every input's final entry, its script at off[i] (exclusive prefix of the lengths) of `scripts`; absent: zero, pad_[0] = 1
__global__ void k_mempool_entries_out(const DevEntry* __restrict__ dent, const uint32_t* __restrict__ off, size_t n, kgv_utxo_entry* __restrict__ out,
                                      uint8_t* __restrict__ scripts) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const DevEntry d = dent[i];
  kgv_utxo_entry e;
  memset(&e, 0, sizeof e);
  e.script_off = off[i];
  if (d.found) {
    e.amount = d.amount; e.block_daa_score = d.block_daa_score; e.script_len = d.script_len; e.spk_version = d.spk_version; e.is_coinbase = d.is_coinbase;
    for (uint32_t k = 0; k < d.script_len; k++) scripts[e.script_off + k] = d.script[k];
  } else {
    e.pad_[0] = 1;
  }
  out[i] = e;
}

// plan: one thread per input. counts[0][i] = Schnorr items, counts[1][i] = ECDSA items (0 when the tx already failed).
__global__ void k_plan(BatchView b, size_t n_inputs, const uint32_t* __restrict__ input_tx, const kgv_tx_result* __restrict__ res,
                       InputPlan* __restrict__ plans, uint32_t* __restrict__ cnt_s, uint32_t* __restrict__ cnt_e) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs) return;
  InputPlan pl;
  pl.item_base = 0; pl.redeem_off = 0; pl.redeem_len = 0; pl.cls = CLS_NONSTANDARD; pl.m = pl.n = pl.n_items = 0; pl.pad_[0] = pl.pad_[1] = 0;
  uint32_t cs = 0, ce = 0;
  if (res[input_tx[i]].status == KGV_TX_OK) {
    const kgv_input& in = b.inputs[i];
    plan_input(pl, b.bytes + in.sigscript_off, in.sigscript_len, b.entries[i]);
    if (pl.cls == CLS_P2PK || pl.cls == CLS_MULTISIG) cs = pl.n_items;
    if (pl.cls == CLS_P2PK_ECDSA || pl.cls == CLS_MULTISIG_ECDSA) ce = pl.n_items;
  }
  plans[i] = pl;
  cnt_s[i] = cs;
  cnt_e[i] = ce;
}

// exclusive scans of the two per-input item-count arrays (Schnorr / ECDSA), one block each in ONE launch: every thread sums a
// contiguous chunk, the 1024 chunk sums are scanned in shared memory, then each thread rewrites its chunk.  (Plumbing: a few
// microseconds for a few hundred thousand inputs; the first version scanned 1024 elements per barrier-laden pass and took
// 80 us per array for a 49 k-input window.)
__global__ void __launch_bounds__(1024) k_exclusive_scan2(const uint32_t* __restrict__ in0, uint32_t* __restrict__ out0, const uint32_t* __restrict__ in1,
                                                          uint32_t* __restrict__ out1, size_t n, uint32_t* __restrict__ totals) {
  const uint32_t* in = blockIdx.x ? in1 : in0;
  uint32_t* out = blockIdx.x ? out1 : out0;
  __shared__ uint32_t part[1024];
  const size_t per = (n + 1023) / 1024;
  const size_t a = (size_t)threadIdx.x * per;
  const size_t b = a + per < n ? a + per : n;
  uint32_t s = 0;
  for (size_t i = a; i < b; i++) s += in[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    uint32_t t = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  uint32_t run = part[threadIdx.x] - s;  // exclusive prefix of this thread's chunk
  for (size_t i = a; i < b; i++) {
    uint32_t v = in[i];
    out[i] = run;
    run += v;
  }
  if (threadIdx.x == 1023) totals[blockIdx.x] = part[1023];
}

// one array (in1 == null: one block) or two, for the other translation units
int kgv_scan_u32(kgv_ctx* ctx, const uint32_t* in0, uint32_t* out0, const uint32_t* in1, uint32_t* out1, size_t n, uint32_t* totals, cudaStream_t st) {
  k_exclusive_scan2<<<in1 ? 2 : 1, 1024, 0, st>>>(in0, out0, in1, out1, n, totals);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

struct ItemRef { uint32_t input; uint32_t k; };  // which input / which candidate pair

__global__ void k_emit_items(BatchView b, size_t n_inputs, InputPlan* __restrict__ plans, const uint32_t* __restrict__ off_s, const uint32_t* __restrict__ off_e,
                             uint8_t* __restrict__ pk_s, uint8_t* __restrict__ sig_s, ItemRef* __restrict__ ref_s,
                             uint8_t* __restrict__ pk_e, uint8_t* __restrict__ sig_e, ItemRef* __restrict__ ref_e) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs) return;
  InputPlan pl = plans[i];
  if (pl.n_items == 0) return;
  bool ecdsa = pl.cls == CLS_P2PK_ECDSA || pl.cls == CLS_MULTISIG_ECDSA;
  uint32_t base = ecdsa ? off_e[i] : off_s[i];
  plans[i].item_base = base;
  const kgv_input& in = b.inputs[i];
  const uint8_t* ss = b.bytes + in.sigscript_off;
  for (uint32_t k = 0; k < pl.n_items; k++) {
    const uint8_t *sig, *key;
    item_location(pl, k, ss, b.entries[i], sig, key);
    size_t it = base + k;
    if (ecdsa) {
      for (int x = 0; x < 33; x++) pk_e[33 * it + x] = key[x];
      for (int x = 0; x < 64; x++) sig_e[64 * it + x] = sig[x];
      ref_e[it] = ItemRef{(uint32_t)i, k};
    } else {
      for (int x = 0; x < 32; x++) pk_s[32 * it + x] = key[x];
      for (int x = 0; x < 64; x++) sig_s[64 * it + x] = sig[x];
      ref_s[it] = ItemRef{(uint32_t)i, k};
    }
  }
}

__global__ void __launch_bounds__(128) k_sighash_reused_v(BatchView b, uint32_t n_txs, const kgv_tx_result* __restrict__ res, SigHashReused* __restrict__ reused) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_txs) return;
  if (res[i].status != KGV_TX_OK) return;
  SigHashReused r;
  sighash_reused(r, b, i);
  reused[i] = r;
}

__global__ void __launch_bounds__(128)
k_item_msgs(BatchView b, const SigHashReused* __restrict__ reused, const uint32_t* __restrict__ input_tx, const InputPlan* __restrict__ plans,
            const ItemRef* __restrict__ refs, size_t n_items, bool ecdsa, uint32_t* __restrict__ msgs) {
  size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= n_items) return;
  ItemRef rf = refs[it];
  InputPlan pl = plans[rf.input];
  const kgv_input& in = b.inputs[rf.input];
  const uint8_t* ss = b.bytes + in.sigscript_off;
  const uint8_t *sig, *key;
  item_location(pl, rf.k, ss, b.entries[rf.input], sig, key);
  uint32_t ht = sig[64];
  uint32_t w[8];
  if (!sighash_type_allowed(ht)) {
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = 0;  // never consulted: resolve reports InvalidSigHashType first
  } else {
    uint32_t tx = input_tx[rf.input];
    SigHashReused r = reused[tx];
    sighash_final(w, b, tx, rf.input, ht, ecdsa, r);
  }
#pragma unroll
  for (int k = 0; k < 8; k++) msgs[8 * it + k] = bswap32(w[k]);
}

__global__ void k_resolve(BatchView b, size_t n_inputs, const uint32_t* __restrict__ input_tx, const kgv_tx_result* __restrict__ res,
                          const InputPlan* __restrict__ plans, const uint8_t* __restrict__ st_s, const uint8_t* __restrict__ st_e,
                          uint8_t* __restrict__ input_err) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs) return;
  if (res[input_tx[i]].status != KGV_TX_OK) { input_err[i] = KGV_SCRIPT_OK; return; }
  InputPlan pl = plans[i];
  const kgv_input& in = b.inputs[i];
  bool ecdsa = pl.cls == CLS_P2PK_ECDSA || pl.cls == CLS_MULTISIG_ECDSA;
  const uint8_t* st = (ecdsa ? st_e : st_s) + pl.item_base;
  input_err[i] = (uint8_t)resolve_input(pl, b.bytes + in.sigscript_off, b.entries[i], in.sig_op_count, st);
}

__global__ void k_tx_finalize(BatchView b, uint32_t n_txs, const uint8_t* __restrict__ input_err, kgv_tx_result* __restrict__ res) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  kgv_tx_result r = res[ti];
  if (r.status != KGV_TX_OK) return;
  const kgv_tx& t = b.txs[ti];
  for (uint32_t i = 0; i < t.n_inputs; i++) {  // check_scripts_sequential order (:170-178)
    uint32_t err = input_err[t.first_input + i];
    if (err == KGV_SCRIPT_OK) continue;
    r.fail_input = i;
    r.script_err = (uint8_t)err;
    if (err == KGV_SCRIPT_NONSTANDARD) r.status = KGV_TX_NEEDS_HOST_VM;
    else r.status = b.inputs[t.first_input + i].sigscript_len == 0 ? KGV_TX_SIGNATURE_EMPTY : KGV_TX_SIGNATURE_INVALID;  // map_script_err :198-200
    break;
  }
  res[ti] = r;
}

__global__ void k_input_tx_index(const kgv_tx* __restrict__ txs, uint32_t n_txs, uint32_t* __restrict__ input_tx) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  kgv_tx t = txs[ti];
  for (uint32_t i = 0; i < t.n_inputs; i++) input_tx[t.first_input + i] = ti;
}

// apply accepted transactions to the table (UtxoDiff::add_transaction, utxo_diff.rs:233-247)
__global__ void k_apply_erase(TableView t, const kgv_tx* __restrict__ txs, const kgv_input* __restrict__ inputs, size_t n_inputs,
                              const uint32_t* __restrict__ input_tx, const uint8_t* __restrict__ accept) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inputs) return;
  if (!accept[input_tx[i]]) return;
  uint32_t k[9];
  input_key(k, inputs[i]);
  table_erase(t, k);
}
__global__ void k_output_tx_index(const kgv_tx* __restrict__ txs, uint32_t n_txs, uint32_t* __restrict__ output_tx) {
  uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= n_txs) return;
  kgv_tx t = txs[ti];
  for (uint32_t i = 0; i < t.n_outputs; i++) output_tx[t.first_output + i] = ti;
}
__global__ void k_apply_insert(TableView t, BatchView b, size_t n_outputs, const uint32_t* __restrict__ output_tx, const uint8_t* __restrict__ accept,
                               const uint64_t* __restrict__ txids, uint64_t pov) {
  size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_outputs) return;
  uint32_t ti = output_tx[o];
  if (!accept[ti]) return;
  const kgv_tx& tx = b.txs[ti];
  const kgv_output& out = b.outputs[o];
  uint32_t k[9];
#pragma unroll
  for (int w = 0; w < 4; w++) { k[2 * w] = (uint32_t)txids[4 * (size_t)ti + w]; k[2 * w + 1] = (uint32_t)(txids[4 * (size_t)ti + w] >> 32); }
  k[8] = (uint32_t)(o - tx.first_output);
  table_put(t, k, out.value, pov, out.spk_version, tx_is_coinbase(tx) ? 1u : 0u, b.bytes + out.script_off, out.script_len);
}

// ---------------------------------------------------------------------------------------------
// K8 MuHash elements (consensus/core/src/muhash.rs:16-33): one element per thread, written straight into level 0
// of its product tree.  Inputs of accepted txs -> denominator tree (the populated entry they spend), outputs ->
// numerator tree (entry = (value, spk, pov_daa_score, tx.is_coinbase)); everything else gets the identity.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_muhash_tx_elements(BatchView b, size_t n_inputs, size_t n_outputs, const uint32_t* __restrict__ input_tx,
                                                            const uint32_t* __restrict__ output_tx, const uint8_t* __restrict__ accept,
                                                            const uint64_t* __restrict__ txids, uint64_t pov, uint32_t* __restrict__ e_den,
                                                            uint32_t* __restrict__ e_num) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_inputs) {
    const uint32_t ti = input_tx[g];
    const DevEntry& e = b.entries[g];
    if (!accept[ti] || !e.found) { u3072_store_one(e_den, n_inputs, g); return; }
    const kgv_input& in = b.inputs[g];
    uint32_t k[8];
#pragma unroll
    for (int w = 0; w < 8; w++)
      k[w] = (uint32_t)in.prev_txid[4 * w] | ((uint32_t)in.prev_txid[4 * w + 1] << 8) | ((uint32_t)in.prev_txid[4 * w + 2] << 16) | ((uint32_t)in.prev_txid[4 * w + 3] << 24);
    uint64_t d[4];
    muhash_utxo_digest(d, k, in.prev_index, e.block_daa_score, e.amount, e.is_coinbase != 0, e.spk_version, e.script, e.script_len);
    muhash_expand_store(e_den, n_inputs, g, d);
    return;
  }
  g -= n_inputs;
  if (g >= n_outputs) return;
  const uint32_t ti = output_tx[g];
  if (!accept[ti]) { u3072_store_one(e_num, n_outputs, g); return; }
  const kgv_tx& tx = b.txs[ti];
  const kgv_output& out = b.outputs[g];
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 4; w++) { k[2 * w] = (uint32_t)txids[4 * (size_t)ti + w]; k[2 * w + 1] = (uint32_t)(txids[4 * (size_t)ti + w] >> 32); }
  uint64_t d[4];
  muhash_utxo_digest(d, k, (uint32_t)(g - tx.first_output), pov, out.value, tx_is_coinbase(tx), out.spk_version, b.bytes + out.script_off, out.script_len);
  muhash_expand_store(e_num, n_outputs, g, d);
}
// live entries of table slots [first, first + n) -> elements (empty slots: identity)
__global__ void __launch_bounds__(128) k_muhash_table_elements(TableView t, uint64_t first, size_t n, uint32_t* __restrict__ e_num) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const UtxoSlot* s = &t.slots[first + g];
  if (s->state != SLOT_FULL) { u3072_store_one(e_num, n, g); return; }
  DevEntry e;
  slot_to_entry(e, t, s);
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = s->key[w];
  uint64_t d[4];
  muhash_utxo_digest(d, k, s->key[8], e.block_daa_score, e.amount, e.is_coinbase != 0, e.spk_version, e.script, e.script_len);
  muhash_expand_store(e_num, n, g, d);
}
// contiguous 384-byte values -> level-0 layout
__global__ void k_u3072_scatter(const uint32_t* __restrict__ values, size_t n, uint32_t* __restrict__ e) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  for (int i = 0; i < KGV_U3072_BLOCKS; i++) u3072_store_block(e, n, g, i, values + 96 * g + 8 * i);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------

extern "C" int kgv_utxo_create(kgv_ctx* ctx, uint64_t capacity_slots, kgv_utxo_table** out) {
  if (!ctx || !out) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  uint64_t cap = 1024;
  while (cap < capacity_slots) cap <<= 1;
  kgv_utxo_table* t = new kgv_utxo_table();
  t->sync = std::make_shared<kgv_table_sync>();
  t->sync->device = ctx->device;
  t->mask = cap - 1;
  t->overflow_cap = cap * 8 < (64ull << 20) ? (64ull << 20) : cap * 8;
  cudaError_t e = cudaMalloc((void**)&t->slots, cap * sizeof(UtxoSlot));
  if (e == cudaSuccess) e = cudaMalloc((void**)&t->overflow, t->overflow_cap);
  if (e == cudaSuccess) e = cudaMalloc((void**)&t->counters, 16 * sizeof(unsigned long long));
  if (e != cudaSuccess) {
    ctx->err = std::string("cudaMalloc failed for the UTXO table: ") + cudaGetErrorString(e);
    (void)cudaGetLastError();
    if (t->slots) cudaFree(t->slots);
    if (t->overflow) cudaFree(t->overflow);
    delete t;
    return KGV_ERR_NOMEM;
  }
  CK(cudaMemsetAsync(t->slots, 0, cap * sizeof(UtxoSlot), ctx->stream));
  CK(cudaMemsetAsync(t->counters, 0, 16 * sizeof(unsigned long long), ctx->stream));
  CK(cudaMalloc((void**)&t->d_view, sizeof(TableView)));
  TableView hv = view_of(t);
  CK(cudaMemcpyAsync(t->d_view, &hv, sizeof hv, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *out = t;
  return KGV_OK;
}

// ---------------------------------------------------------------------------------------------
// composed views: a diff layer on the device (utxo_view.rs:22-35, utxo_diff.rs:15-19)
// ---------------------------------------------------------------------------------------------
extern "C" int kgv_utxo_view_create(kgv_ctx* ctx, kgv_utxo_table* base, uint64_t capacity_slots, kgv_utxo_table** out) {
  if (!ctx || !base || !out) return KGV_ERR_ARG;
  if (base->sync->device != ctx->device) {
    std::lock_guard<std::recursive_mutex> g(ctx->mu);
    ctx->err = "kgv_utxo_view_create: the base table belongs to device " + std::to_string(base->sync->device) + ", the context to device " + std::to_string(ctx->device);
    return KGV_ERR_ARG;
  }
  int rc = kgv_utxo_create(ctx, capacity_slots, out);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  (*out)->base = base;
  TableView hv = view_of(*out);  // now with `below`
  CK(cudaMemcpyAsync((*out)->d_view, &hv, sizeof hv, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}
// write_diff_batch (utxo_set.rs:107-112): delete what the layer removed, put what it added - applied to the layer below through that layer's own
// view semantics (so a stack of diffs folds downwards one level at a time)
__global__ void k_view_commit_removes(TableView top, TableView below) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > top.mask) return;
  const UtxoSlot* s = &top.slots[i];
  const uint32_t st = s->state;
  if (st != SLOT_REMOVED && st != SLOT_FULLH) return;
  uint32_t k[9];
#pragma unroll
  for (int w = 0; w < 9; w++) k[w] = s->key[w];
  table_erase(below, k);
}
__global__ void k_view_commit_adds(TableView top, TableView below) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > top.mask) return;
  const UtxoSlot* s = &top.slots[i];
  const uint32_t st = s->state;
  if (st != SLOT_FULL && st != SLOT_FULLH) return;
  SlotHead h;
  slot_load_head(h, s);
  DevEntry e;
  TableView solo = top;
  solo.below = nullptr;
  head_to_entry(e, solo, s, h);
  uint32_t k[9];
#pragma unroll
  for (int w = 0; w < 9; w++) k[w] = s->key[w];
  table_put(below, k, e.amount, e.block_daa_score, e.spk_version, e.is_coinbase, e.script, e.script_len);
}
static int view_clear(kgv_ctx* ctx, kgv_utxo_table* v) {
  CK(cudaMemsetAsync(v->slots, 0, (v->mask + 1) * sizeof(UtxoSlot), ctx->stream));
  CK(cudaMemsetAsync(v->counters, 0, 16 * sizeof(unsigned long long), ctx->stream));
  v->occ_bound = v->arena_bound = 0;
  return KGV_OK;
}
extern "C" int kgv_utxo_view_commit(kgv_ctx* ctx, kgv_utxo_table* view) {
  if (!ctx || !view || !view->base) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);  // reads the layer, writes the base
  if (int rc = acc.acquire("kgv_utxo_view_commit", view, view->base)) return rc;
  if (view->base->max_load) {  // the base takes at most the layer's entries and its long scripts
    unsigned long long c[3];
    CK(cudaMemcpyAsync(c, view->counters, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    int rc = utxo_reserve(ctx, view->base, c[0], c[2]);
    if (rc) return rc;
  }
  TableView top = view_of(view), below = view_of(view->base);
  k_view_commit_removes<<<nblk(view->mask + 1, 128), 128, 0, ctx->stream>>>(top, below);
  CK(cudaGetLastError());
  k_view_commit_adds<<<nblk(view->mask + 1, 128), 128, 0, ctx->stream>>>(top, below);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return view_clear(ctx, view);
}
extern "C" int kgv_utxo_view_discard(kgv_ctx* ctx, kgv_utxo_table* view) {
  if (!ctx || !view || !view->base) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_view_discard", view, view)) return rc;
  return view_clear(ctx, view);
}
// A write like any other: it waits for the open reads and writes of every context, then for their work on the GPU, and frees the table's
// arrays, those retired by earlier rehashes included.
extern "C" void kgv_utxo_destroy(kgv_ctx* ctx, kgv_utxo_table* t) {
  if (!t) return;
  kgv_table_sync* s = t->sync.get();
  cudaSetDevice(s->device);
  if (ctx) cudaStreamSynchronize(ctx->stream);
  {
    std::unique_lock<std::mutex> g(s->m);
    const uint64_t ticket = s->next_ticket++;
    s->cv.wait(g, [&] { return s->serving == ticket && s->write_depth == 0 && s->readers.empty(); });
    for (const auto& r : s->reads) cudaEventSynchronize(r.second);
    if (s->last_write) cudaEventSynchronize(s->last_write);
    for (const auto& r : s->retired) {
      cudaEventSynchronize(r.done);
      for (void* p : r.ptrs) cudaFree(p);
      s->pool.push_back(r.done);
    }
    s->retired.clear();
    for (const auto& r : s->reads) s->pool.push_back(r.second);
    s->reads.clear();
    if (s->last_write) s->pool.push_back(s->last_write);
    s->last_write = nullptr;
    for (cudaEvent_t e : s->pool) cudaEventDestroy(e);
    s->pool.clear();
    s->serving++;
  }
  cudaFree(t->slots); cudaFree(t->overflow); cudaFree(t->counters);
  if (t->d_view) cudaFree(t->d_view);
  delete t;
}

extern "C" int kgv_utxo_lookup(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* keys36, size_t n, kgv_utxo_entry* entries, uint8_t* scripts_out,
                               uint32_t script_stride, uint8_t* found) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!keys36 || !entries || !found || (script_stride && !scripts_out)) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_lookup", t)) return rc;
  kgv_io io(ctx);
  const uint8_t* dk;
  kgv_utxo_entry* de;
  uint8_t *ds, *df;
  io.in(keys36, n * 36, &dk);
  io.out(entries, n * sizeof(kgv_utxo_entry), &de);
  io.inout(script_stride ? scripts_out : nullptr, n * (size_t)script_stride, &ds);  // only each script's bytes are written: the rest stays the caller's
  io.out(found, n, &df);
  if (int rc = io.stage()) return rc;
  k_utxo_lookup<<<nblk(n, 128), 128, 0, ctx->stream>>>(view_of(t), dk, n, de, ds, script_stride, df);
  CK(cudaGetLastError());
  ctx->launches++;
  return io.finish();
}

extern "C" int kgv_utxo_apply_diff(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* rem_keys36, size_t n_rem, uint8_t* rem_status,
                                   const uint8_t* add_keys36, const kgv_utxo_entry* add_entries, const uint8_t* add_bytes, size_t n_add_bytes, size_t n_add,
                                   uint8_t* add_status) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if ((n_rem && !rem_keys36) || (n_add && (!add_keys36 || !add_entries || (n_add_bytes && !add_bytes)))) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  const void* probe = n_rem ? (const void*)rem_keys36 : (const void*)add_keys36;
  if (!probe) return KGV_OK;
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_apply_diff", t, t)) return rc;
  {  // a view layer records a removal marker for an entry that lives below
    int rc = utxo_reserve(ctx, t, n_add + (t->base ? n_rem : 0), n_add_bytes + 8 * (uint64_t)n_add);
    if (rc) return rc;
  }
  kgv_io io(ctx);
  const uint8_t *drk, *dak, *dab;
  const kgv_utxo_entry* dae;
  uint8_t *drs, *das;
  io.in(n_rem ? rem_keys36 : nullptr, n_rem * 36, &drk);
  io.out(n_rem ? rem_status : nullptr, n_rem, &drs);
  io.in(n_add ? add_keys36 : nullptr, n_add * 36, &dak);
  io.in(n_add ? add_entries : nullptr, n_add * sizeof(kgv_utxo_entry), &dae);
  io.in(n_add && n_add_bytes ? add_bytes : nullptr, n_add_bytes, &dab);
  io.out(n_add ? add_status : nullptr, n_add, &das);
  if (int rc = io.stage()) return rc;
  if (n_rem) { k_utxo_erase<<<nblk(n_rem, 128), 128, 0, ctx->stream>>>(view_of(t), drk, n_rem, drs); CK(cudaGetLastError()); ctx->launches++; }
  if (n_add) { k_utxo_insert<<<nblk(n_add, 128), 128, 0, ctx->stream>>>(view_of(t), dak, dae, dab, n_add, das); CK(cudaGetLastError()); ctx->launches++; }
  return io.finish();
}

extern "C" int kgv_utxo_export(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t* keys36, kgv_utxo_entry* entries, uint8_t* bytes, size_t max_n, size_t bytes_cap, size_t* n_out,
                               size_t* bytes_out) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (t->base) { ctx->err = "export is defined on plain tables: commit the view first"; return KGV_ERR_ARG; }
  const bool counting = !keys36;
  if (!counting && (!entries || (bytes_cap && !bytes))) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"n_out", n_out}, {"bytes_out", bytes_out}})
    if (int rc = kgv_host_only(ctx, "kgv_utxo_export", what, p)) return rc;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_export", t)) return rc;
  kgv_io io(ctx);
  uint8_t *dk = nullptr, *db = bytes;
  kgv_utxo_entry* de = entries;
  if (!counting) {
    io.out(keys36, max_n * 36, &dk);
    io.out(entries, max_n * sizeof(kgv_utxo_entry), &de);
    io.out(bytes, bytes_cap, &db);
    if (int rc = io.stage()) return rc;
  }
  // the counts live in the context's scratch: other contexts may export the table at the same time
  if (int rc = kgv_reserve(ctx, &ctx->d_work, &ctx->d_work_cap, 2 * sizeof(unsigned long long))) return rc;
  unsigned long long* cnt = (unsigned long long*)ctx->d_work;
  CK(cudaMemsetAsync(cnt, 0, 2 * sizeof(unsigned long long), ctx->stream));
  k_utxo_export<<<nblk(t->mask + 1, 128), 128, 0, ctx->stream>>>(view_of(t), dk, de, db, max_n, bytes_cap, cnt);
  CK(cudaGetLastError());
  ctx->launches++;
  unsigned long long c[2];
  CK(cudaMemcpyAsync(c, cnt, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (n_out) *n_out = (size_t)c[0];
  if (bytes_out) *bytes_out = (size_t)c[1];
  if (counting) return KGV_OK;
  if (c[0] > max_n || c[1] > bytes_cap) { ctx->err = "kgv_utxo_export: the caller's arrays are too small (sizes returned)"; return KGV_ERR_NOMEM; }
  // only what the table held comes back
  io.trim(keys36, (size_t)c[0] * 36);
  io.trim(entries, (size_t)c[0] * sizeof(kgv_utxo_entry));
  io.trim(bytes, (size_t)c[1]);
  return io.finish();
}

extern "C" int kgv_utxo_import_chunk(kgv_ctx* ctx, kgv_utxo_table* t, const uint8_t* keys36, const kgv_utxo_entry* entries, const uint8_t* bytes, size_t n_bytes, size_t n,
                                     uint8_t* numerator384) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!numerator384) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (n == 0) return KGV_OK;
  if (!keys36 || !entries || (n_bytes && !bytes)) { ctx->err = "null buffer"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_utxo_import_chunk", "numerator384", numerator384)) return rc;
  kgv_io io(ctx);
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_import_chunk", t, t)) return rc;
  // the script ranges are checked here whatever the side of entries: device entries are read through a host copy
  std::vector<kgv_utxo_entry> entries_host;
  const kgv_utxo_entry* he = entries;
  if (io.is_device(entries)) {
    entries_host.resize(n);
    CK(cudaMemcpyAsync(entries_host.data(), entries, n * sizeof(kgv_utxo_entry), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    he = entries_host.data();
  }
  for (size_t i = 0; i < n; i++)
    if ((uint64_t)he[i].script_off + he[i].script_len > n_bytes) { ctx->err = "kgv_utxo_import_chunk: entry script outside the byte arena"; return KGV_ERR_ARG; }
  // one upload serves the insert and the multiset
  const uint8_t *dk, *db;
  const kgv_utxo_entry* de;
  io.in(keys36, n * 36, &dk);
  io.in(entries, n * sizeof(kgv_utxo_entry), &de);
  io.in(n_bytes ? bytes : nullptr, n_bytes, &db);
  if (int rc = io.stage()) return rc;
  // pruning_meta.utxo_set.write_many(chunk) (consensus/mod.rs:1072)
  int rc = kgv_utxo_apply_diff(ctx, t, nullptr, 0, nullptr, dk, de, db, n_bytes, n, nullptr);
  if (rc) return rc;
  // chunk.par_iter().map(MuHash::from_utxo).reduce(combine) (:1075-1080), then current_multiset.combine (:1082)
  uint32_t *e_den = nullptr, *e_num = nullptr;
  rc = kgv_mu_reserve(ctx, 0, n, &e_den, &e_num);
  if (rc) return rc;
  k_muhash_utxo_elements<<<nblk(n, 128), 128, 0, ctx->stream>>>(dk, de, db, n, e_num);
  CK(cudaGetLastError());
  ctx->launches++;
  uint8_t chunk_num[384], chunk_den[384], one[384];
  rc = kgv_mu_reduce(ctx, io, 0, n, chunk_num, chunk_den);
  if (rc) return rc;
  memset(one, 0, sizeof one);
  one[0] = 1;
  uint8_t den[384];
  memcpy(den, one, sizeof den);
  return kgv_muhash_combine(ctx, numerator384, den, chunk_num, one);
}

extern "C" int kgv_utxo_count(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t* count) {
  if (!ctx || !t || !count) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (int rc = kgv_host_only(ctx, "kgv_utxo_count", "count", count)) return rc;
  if (t->base) { ctx->err = "count / digest / MuHash are defined on plain tables: commit the view first"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_count", t)) return rc;
  unsigned long long c[4];
  CK(cudaMemcpyAsync(c, t->counters, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (c[3]) { ctx->err = "UTXO table insert failures (table or overflow arena full)"; return KGV_ERR_NOMEM; }
  *count = c[0];
  return KGV_OK;
}

extern "C" int kgv_utxo_digest(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t out32[32]) {
  if (!ctx || !t || !out32) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (int rc = kgv_host_only(ctx, "kgv_utxo_digest", "out32", out32)) return rc;
  if (t->base) { ctx->err = "count / digest / MuHash are defined on plain tables: commit the view first"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access access(ctx);
  if (int rc = access.acquire("kgv_utxo_digest", t)) return rc;
  // the sums live in the context's scratch: other contexts may digest the table at the same time
  if (int rc = kgv_reserve(ctx, &ctx->d_work, &ctx->d_work_cap, 8 * sizeof(unsigned long long))) return rc;
  unsigned long long* acc = (unsigned long long*)ctx->d_work;
  CK(cudaMemsetAsync(acc, 0, 8 * sizeof(unsigned long long), ctx->stream));
  k_utxo_digest<<<nblk(t->mask + 1, 128), 128, 0, ctx->stream>>>(view_of(t), acc);
  CK(cudaGetLastError());
  ctx->launches++;
  unsigned long long h[8];
  CK(cudaMemcpyAsync(h, acc, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  unsigned __int128 c = 0;
  for (int i = 0; i < 8; i++) {  // fold the 32-bit limb sums into a 256-bit little-endian integer (mod 2^256)
    c += h[i];
    uint32_t limb = (uint32_t)c;
    c >>= 32;
    for (int b = 0; b < 4; b++) out32[4 * i + b] = (uint8_t)(limb >> (8 * b));
  }
  return KGV_OK;
}

// The verification step of a list of items on stream s: without a SigCache every item is verified; with one, hits are answered from the
// table and only the misses are verified (and remembered).  dig / idx / nm: the cache's digests, miss list and miss count (unused without).
int kgv_verify_items(kgv_ctx* ctx, kgv_sigcache* sc, const uint8_t* pk, const uint8_t* msg, const uint8_t* sig, size_t n, bool ecdsa, uint8_t* st, uint8_t* dig,
                     uint32_t* idx, uint32_t* nm, cudaStream_t s) {
  if (!sc) return kgv_launch_verify(ctx, pk, msg, sig, n, st, ecdsa, s);
  int r = kgv_sigcache_lookup(ctx, sc, pk, msg, sig, n, ecdsa, st, dig, idx, nm, s);
  if (!r) r = kgv_launch_verify(ctx, pk, msg, sig, n, st, ecdsa, s, idx, nm);
  if (!r) r = kgv_sigcache_insert(ctx, sc, st, dig, idx, nm, n, s);
  return r;
}

// The script phase of check_scripts (tx_validation_in_utxo_context.rs:162-200) for every transaction whose dres[].status is
// KGV_TX_OK: plan -> scan -> emit -> sighash -> verify -> resolve -> finalize, all enqueued on ctx->stream (the ECDSA items on
// the side stream).  v.entries must be populated.  Uses ctx->d_scratch (plans, counts, offsets, sub-hashes) and ctx->d_in
// (item arrays); one host synchronisation (the two item totals).
int kgv_scripts_phase(kgv_ctx* ctx, const BatchView& v, size_t nt, size_t ni, const uint32_t* itx, kgv_tx_result* dres, uint64_t* n_items_out) {
  if (n_items_out) *n_items_out = 0;
  if (ni == 0) return KGV_OK;
  InputPlan* plans;
  uint32_t *cs, *ce, *os, *oe, *tot;
  uint8_t* ierr;
  SigHashReused* reu;
  int rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap, [&](kgv_carve& c) {
    plans = c.take<InputPlan>(ni);
    cs = c.take<uint32_t>(ni); ce = c.take<uint32_t>(ni); os = c.take<uint32_t>(ni); oe = c.take<uint32_t>(ni); tot = c.take<uint32_t>(16);
    ierr = c.take<uint8_t>(ni); reu = c.take<SigHashReused>(nt);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  k_plan<<<nblk(ni, 128), 128, 0, st>>>(v, ni, itx, dres, plans, cs, ce);
  CK(cudaGetLastError());
  STAGE("plan");
  k_exclusive_scan2<<<2, 1024, 0, st>>>(cs, os, ce, oe, ni, tot);
  CK(cudaGetLastError());
  ctx->launches += 2;
  uint32_t totals[2];
  CK(cudaMemcpyAsync(totals, tot, sizeof totals, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  size_t ns = totals[0], ne = totals[1];
  if (n_items_out) *n_items_out = ns + ne;
  if (kgv_debug_on()) fprintf(stderr, "[kgv] items: schnorr %zu ecdsa %zu\n", ns, ne);
  // multi-GPU (kgv_set_sharding): the candidate pairs of each kind are split into n_ranks contiguous ranges; this rank verifies one and
  // the status bytes are exchanged before the scripts are resolved
  int nr = 1, rk = 0;
  if (ctx->shard_comm) nr = kgv_comm_ranks(ctx->shard_comm, &rk);
  // signature cache (kgv_set_sigcache; not combined with sharding)
  kgv_sigcache* sc = nr == 1 ? ctx->sigcache : nullptr;
  // item arrays of the two kinds ([0] Schnorr, [1] ECDSA) in d_in: pk, sig, msg, refs, status (padded to nr * per), and with the signature
  // cache the digests, the miss list and the miss count
  struct ItemKind {
    size_t n, per, lo, hi;  // items, range length per rank, this rank's range [lo, hi)
    uint8_t *pk, *sig, *msg, *st, *dig;  // the item arrays in d_in
    ItemRef* ref;
    uint32_t *idx, *nm;
  } kind[2];
  for (int e = 0; e < 2; e++) {
    ItemKind& k = kind[e];
    k.n = e ? ne : ns;
    k.per = nr > 1 ? al256((k.n + nr - 1) / nr) : k.n;
    k.lo = std::min(rk * k.per, k.n);
    k.hi = std::min((rk + 1) * k.per, k.n);
  }
  rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) {
    for (int e = 0; e < 2; e++) {
      ItemKind& k = kind[e];
      k.pk = c.take<uint8_t>(k.n * (e ? 33 : 32)); k.sig = c.take<uint8_t>(k.n * 64); k.msg = c.take<uint8_t>(k.n * 32); k.ref = c.take<ItemRef>(k.n);
      k.st = c.take<uint8_t>(nr * k.per, 64);
      k.dig = c.take<uint8_t>(sc ? k.n * 32 : 0); k.idx = c.take<uint32_t>(sc ? k.n : 0); k.nm = c.take<uint32_t>(16);
    }
  });
  if (rc) return rc;
  if (ns + ne) {
    k_emit_items<<<nblk(ni, 128), 128, 0, st>>>(v, ni, plans, os, oe, kind[0].pk, kind[0].sig, kind[0].ref, kind[1].pk, kind[1].sig, kind[1].ref);
    CK(cudaGetLastError());
    k_sighash_reused_v<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, dres, reu);
    CK(cudaGetLastError());
    ctx->launches += 2;
    STAGE("emit+reused");
  }
  // one kind's messages and verdicts on stream s, for this rank's range
  auto verify_kind = [&](bool ecdsa, cudaStream_t s) -> int {
    const ItemKind& k = kind[ecdsa];
    if (k.hi <= k.lo) return KGV_OK;
    const size_t m = k.hi - k.lo;
    k_item_msgs<<<nblk(m, 128), 128, 0, s>>>(v, reu, itx, plans, k.ref + k.lo, m, ecdsa, (uint32_t*)k.msg + 8 * k.lo);
    CK(cudaGetLastError());
    ctx->launches++;
    STAGE(ecdsa ? "msgs ecdsa" : "msgs schnorr");
    // (with the cache there is one rank: lo = 0, m = n)
    return kgv_verify_items(ctx, sc, k.pk + (ecdsa ? 33 : 32) * k.lo, k.msg + 32 * k.lo, k.sig + 64 * k.lo, m, ecdsa, k.st + k.lo, k.dig, k.idx, k.nm, s);
  };
  if (ns && ne) CK(cudaEventRecord(ctx->ev_fork, st));  // fork point: everything both item kinds depend on is queued
  if (ns) {
    rc = verify_kind(false, st);
    if (rc) return rc;
    STAGE("verify schnorr");
  }
  if (ne) {
    // with both kinds present the ECDSA items run on the side stream so the two (often sub-wave) verify
    // launches share the SMs instead of queueing behind each other
    const bool fork = ns != 0 && !kgv_debug_on();
    cudaStream_t se = fork ? ctx->aux_stream : st;
    if (fork) CK(cudaStreamWaitEvent(se, ctx->ev_fork, 0));
    rc = verify_kind(true, se);
    if (rc) return rc;
    if (fork) {
      CK(cudaEventRecord(ctx->ev_join, se));
      CK(cudaStreamWaitEvent(st, ctx->ev_join, 0));
    }
    STAGE("verify ecdsa");
  }
  if (nr > 1) {
    for (const ItemKind& k : kind)
      if (k.n) { rc = kgv_comm_exchange_slices(ctx, ctx->shard_comm, k.st, k.per); if (rc) return rc; }
    STAGE("verdict exchange");
  }
  k_resolve<<<nblk(ni, 128), 128, 0, st>>>(v, ni, itx, dres, plans, kind[0].st, kind[1].st, ierr);
  CK(cudaGetLastError());
  STAGE("resolve");
  k_tx_finalize<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, ierr, dres);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return KGV_OK;
}

__global__ void k_count_status(const kgv_tx_result* __restrict__ res, uint32_t n, uint8_t what, unsigned long long* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = i < n && res[i].status == what;
  unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(out, (unsigned long long)__popc(m));
}

// The script phase of a validation call against a table (kgv_validate_txs, kgv_validate_mempool_txs), then the device script engine for what
// it declined: utxo_validation.rs:282-309 accepts ANY transaction whose scripts execute successfully, so a non-standard spend must not leave
// the call undecided.  The engine runs on the entries the call populated (v.entries), long scripts in the table's overflow arena included.
// cnt: one u64 of device scratch of the call (not of the table, which other contexts may be reading at the same time).
static int scripts_with_engine(kgv_ctx* ctx, unsigned long long* cnt, const kgv_dev_batch& d, const BatchView& v, const uint32_t* itx, kgv_tx_result* dres) {
  const size_t nt = d.n_txs;
  int rc = kgv_scripts_phase(ctx, v, nt, d.n_inputs, itx, dres, nullptr);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  unsigned long long n_vm = 0;
  CK(cudaMemsetAsync(cnt, 0, 8, st));
  k_count_status<<<nblk(nt, 256), 256, 0, st>>>(dres, (uint32_t)nt, KGV_TX_NEEDS_HOST_VM, cnt);
  CK(cudaGetLastError());
  ctx->launches++;
  CK(cudaMemcpyAsync(&n_vm, cnt, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return n_vm ? kgv_script_engine_run(ctx, v, nt, nullptr, (size_t)n_vm, dres, true, nullptr) : KGV_OK;
}

// shared core of kgv_validate_populated / kgv_validate_txs
static int validate_core(kgv_ctx* ctx, kgv_utxo_table* table, const kgv_tx_batch* batch, uint64_t pov, uint32_t flags, const kgv_params* prm,
                         kgv_tx_result* results) {
  if (!batch || !prm || (batch->n_txs && !results)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (flags > KGV_FLAGS_SCRIPTS_ONLY) { ctx->err = "unknown validation flags"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, table ? "kgv_validate_txs" : "kgv_validate_populated", "params", prm)) return rc;
  if (batch->n_txs == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (table)
    if (int rc = acc.acquire("kgv_validate_txs", table)) return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, table == nullptr);
  if (rc) return rc;
  const size_t nt = d.n_txs, ni = d.n_inputs;
  DevEntry* dent;
  uint32_t* itx;
  kgv_tx_result* dres;
  unsigned long long* cnt;
  rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) {
    dent = c.take<DevEntry>(ni); itx = c.take<uint32_t>(ni); dres = c.take<kgv_tx_result>(nt); cnt = c.take<unsigned long long>(1);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;

  if (ni) {
    if (table) k_populate<<<nblk(ni, 128), 128, 0, st>>>(view_of(table), d.inputs, ni, dent);
    else k_entries_from_batch<<<nblk(ni, 128), 128, 0, st>>>(d.entries, d.bytes, ni, dent);
    CK(cudaGetLastError());
    k_input_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, itx);
    CK(cudaGetLastError());
    ctx->launches += 2;
  }
  STAGE("populate");
  BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
  k_tx_context<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, pov, flags, *prm, dres);
  CK(cudaGetLastError());
  ctx->launches++;
  STAGE("tx_context");
  if (flags != KGV_FLAGS_SKIP_SCRIPT_CHECKS && ni) {
    rc = table ? scripts_with_engine(ctx, cnt, d, v, itx, dres) : kgv_scripts_phase(ctx, v, nt, ni, itx, dres, nullptr);
    if (rc) return rc;
  }
  kgv_io io(ctx);
  if ((rc = io.copy_out(results, dres, nt * sizeof(kgv_tx_result)))) return rc;
  return io.finish();
}

extern "C" int kgv_validate_populated(kgv_ctx* ctx, const kgv_tx_batch* batch, uint64_t pov_daa_score, uint32_t flags, const kgv_params* params,
                                      kgv_tx_result* results) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  return validate_core(ctx, nullptr, batch, pov_daa_score, flags, params, results);
}
extern "C" int kgv_validate_txs(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t pov_daa_score, uint32_t flags, const kgv_params* params,
                                kgv_tx_result* results) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  return validate_core(ctx, t, batch, pov_daa_score, flags, params, results);
}

// validate_mempool_transaction_in_utxo_context for a batch (utxo_validation.rs:341-397): populate (caller's entries first), the mempool rule
// order with the storage mass computed and the feerate threshold (k_tx_mempool_context), the final entries written out, then the script phase
// of kgv_validate_txs.  The entries go out BEFORE the script phase, so a too small scripts_out is reported before any signature is verified.
// One synchronisation before the script phase reads the script bytes and the zero-divisor count.
// iso (kgv_validate_mempool_txs_in_parallel): the isolation and finality rules run first, on the device; their verdicts gate the lookups
// and the context rules, and their masses replace args[i].non_contextual_mass.  iso == null is kgv_validate_mempool_txs.
// iso->policy (kgv_validate_mempool_txs_with_policy): standardness in isolation right after the isolation rules (its failures override
// the gate) and standardness in context after the scripts, for the txs still KGV_TX_OK.
struct MempoolIso {
  const kgv_tx_rules* rules;
  uint64_t past_median_time;
  kgv_tx_masses* masses;                     // caller's output, may be null
  const kgv_mempool_policy* policy = nullptr;
  uint64_t* detail = nullptr;                // caller's output, may be null
};
static int mempool_core(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t virtual_daa_score, const kgv_params* prm,
                        const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_utxo_entry* entries_out,
                        uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used, const MempoolIso* iso) {
  const char* call = !iso ? "kgv_validate_mempool_txs" : iso->policy ? "kgv_validate_mempool_txs_with_policy" : "kgv_validate_mempool_txs_in_parallel";
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"params", prm}, {"rules", iso ? iso->rules : nullptr},
                                {"policy", iso ? iso->policy : nullptr}, {"scripts_used", scripts_used}})
    if (int rc = kgv_host_only(ctx, call, what, p)) return rc;
  if (scripts_used) *scripts_used = 0;
  if (!batch || !prm || (batch->n_txs && (!results || !storage_mass)) || (entries_out && scripts_cap && !scripts_out) || (iso && !iso->rules)) {
    ctx->err = "null argument";
    return KGV_ERR_ARG;
  }
  if (batch->n_txs == 0) return KGV_OK;
  if (iso && batch->n_txs > 0xFFFFFFFFull) { ctx->err = "kgv_validate_mempool_txs_in_parallel: more than 2^32 - 1 transactions"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  // one read of the table for the three mempool calls, over the whole call: kernels enqueued after its host synchronisations still read it
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire(call, t)) return rc;
  kgv_io io(ctx);
  bool dev;
  if (int rc = io.one_side(call, {results, batch->txs, args, storage_mass, entries_out, scripts_cap ? scripts_out : nullptr,
                                                        iso ? iso->masses : nullptr, iso ? iso->detail : nullptr}, &dev))
    return rc;
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  const size_t nt = d.n_txs, ni = d.n_inputs;
  // d_work: populated entries, input -> tx, verdicts, masses, script lengths and their offsets,
  // counters [script bytes (64-bit), zero divisors, the scan's 32-bit total, the relay-fee overflow flag of the standardness policy, the
  // script engine's count]
  // with iso: its verdicts, max(compute, transient) per tx, the masses (for the policy when the caller takes none), the large-transaction list
  const kgv_mempool_policy* pol = iso ? iso->policy : nullptr;
  uint64_t* detail = iso ? iso->detail : nullptr;
  const bool own_masses = iso && !iso->masses && pol;
  DevEntry* dent;
  uint32_t *itx, *len, *off, *lst;
  kgv_tx_result *dres, *gate;
  uint64_t *dmass, *dnc;
  unsigned long long* cnt;
  kgv_tx_masses* own;
  rc = kgv_reserve_carved(ctx, &ctx->d_work, &ctx->d_work_cap, [&](kgv_carve& c) {
    dent = c.take<DevEntry>(ni); itx = c.take<uint32_t>(ni); dres = c.take<kgv_tx_result>(nt); dmass = c.take<uint64_t>(nt);
    len = c.take<uint32_t>(ni); off = c.take<uint32_t>(ni); cnt = c.take<unsigned long long>(5);
    gate = iso ? c.take<kgv_tx_result>(nt) : nullptr; dnc = iso ? c.take<uint64_t>(nt) : nullptr;
    own = own_masses ? c.take<kgv_tx_masses>(nt) : nullptr; lst = iso ? c.take<uint32_t>(nt + 1) : nullptr;
  });
  if (rc) return rc;
  // the entries' scripts come back up to their size, known after the context rules
  const kgv_mempool_tx_args* dargs;
  kgv_tx_masses* dism = nullptr;
  uint64_t* ddet;
  kgv_utxo_entry* de;
  uint8_t* ds;
  io.in(args, nt * sizeof(kgv_mempool_tx_args), &dargs);
  if (iso) io.out(iso->masses, nt * sizeof(kgv_tx_masses), &dism);
  io.out(pol ? detail : nullptr, nt * 8, &ddet);
  io.out(ni ? entries_out : nullptr, ni * sizeof(kgv_utxo_entry), &de);
  io.out(ni && entries_out && scripts_cap ? scripts_out : nullptr, scripts_cap, &ds);
  if ((rc = io.stage())) return rc;
  cudaStream_t st = ctx->stream;
  CK(cudaMemsetAsync(cnt, 0, 32, st));
  if (iso) {
    if (own_masses) dism = own;
    rc = kgv_isolation_run(ctx, d, *iso->rules, virtual_daa_score, iso->past_median_time, true, gate, dism, dnc, lst, st);
    if (rc) return rc;
    STAGE("isolation");
    if (pol) {
      // the mempool checks standardness in isolation before consensus validates the tx: its failures take the gate's place
      if ((rc = kgv_standard_isolation_run(ctx, d, *pol, dism, true, gate, ddet, st))) return rc;
      STAGE("standard in isolation");
    } else if (detail) {
      if (dev) CK(cudaMemsetAsync(detail, 0, nt * 8, st));
      else memset(detail, 0, nt * 8);
    }
  }
  if (ni) {
    k_input_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, itx);
    CK(cudaGetLastError());
    k_populate_mempool<<<nblk(ni, 128), 128, 0, st>>>(view_of(t), d.inputs, d.entries, d.bytes, ni, dent, len, cnt, gate, itx);
    CK(cudaGetLastError());
    k_exclusive_scan2<<<1, 1024, 0, st>>>(len, off, nullptr, nullptr, ni, (uint32_t*)(cnt + 2));  // block 0 only: one array
    CK(cudaGetLastError());
    ctx->launches += 3;
  }
  STAGE("populate");
  BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
  k_tx_mempool_context<<<nblk(nt, 128), 128, 0, st>>>(v, (uint32_t)nt, virtual_daa_score, *prm, dargs, dres, dmass, cnt + 1, gate, dnc);
  CK(cudaGetLastError());
  ctx->launches++;
  STAGE("mempool context");
  unsigned long long c[2];
  CK(cudaMemcpyAsync(c, cnt, sizeof c, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint64_t n_script = c[0];
  if (scripts_used) *scripts_used = (size_t)n_script;
  if (c[1]) { ctx->err = "kgv_validate_mempool_txs: a feerate threshold with max(storage mass, non_contextual_mass) == 0"; return KGV_ERR_ARG; }
  if (entries_out && n_script > 0xFFFFFFFFull) { ctx->err = "kgv_validate_mempool_txs: the entries' scripts exceed the 32-bit script_off range"; return KGV_ERR_ARG; }
  if (entries_out && n_script > scripts_cap) { ctx->err = "kgv_validate_mempool_txs: scripts_out is too small (size returned)"; return KGV_ERR_NOMEM; }
  if (entries_out && ni) {
    k_mempool_entries_out<<<nblk(ni, 128), 128, 0, st>>>(dent, off, ni, de, ds);
    CK(cudaGetLastError());
    ctx->launches++;
    io.trim(scripts_out, n_script);
  }
  if (ni) {
    rc = scripts_with_engine(ctx, cnt + 4, d, v, itx, dres);
    if (rc) return rc;
  }
  unsigned long long* fee_overflow = cnt + 3;
  if (pol) {
    if ((rc = kgv_standard_context_run(ctx, d, dent, *pol, dism, dmass, nullptr, dres, ddet, fee_overflow, st))) return rc;
    STAGE("standard in context");
  }
  if ((rc = io.copy_out(results, dres, nt * sizeof(kgv_tx_result))) || (rc = io.copy_out(storage_mass, dmass, nt * 8))) return rc;
  // the compute mass of a tx that reaches the fee check is at most 100 000 (standardness in isolation), so only a relay fee above
  // u64::MAX / 100 000 can overflow: a device-pointer caller waits for the flag only then
  unsigned long long overflow = 0;
  if (pol && (!dev || pol->minimum_relay_transaction_fee > ~0ull / kgv::STD_MAX_TRANSACTION_MASS) && (rc = io.copy_out(&overflow, fee_overflow, 8))) return rc;
  if ((rc = io.finish())) return rc;
  if (overflow) { ctx->err = "kgv_validate_mempool_txs_with_policy: compute mass * minimum_relay_transaction_fee overflows u64"; return KGV_ERR_ARG; }
  return KGV_OK;
}

extern "C" int kgv_validate_mempool_txs(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t virtual_daa_score, const kgv_params* prm,
                                        const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_utxo_entry* entries_out,
                                        uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  return mempool_core(ctx, t, batch, virtual_daa_score, prm, args, results, storage_mass, entries_out, scripts_out, scripts_cap, scripts_used, nullptr);
}

// validate_mempool_transaction_impl (processor.rs:823-839) for a batch: isolation -> finality -> the UTXO-context pipeline above
extern "C" int kgv_validate_mempool_txs_in_parallel(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t virtual_daa_score,
                                                    uint64_t virtual_past_median_time, const kgv_params* prm, const kgv_tx_rules* rules,
                                                    const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_tx_masses* masses,
                                                    kgv_utxo_entry* entries_out, uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  const MempoolIso iso{rules, virtual_past_median_time, masses};
  return mempool_core(ctx, t, batch, virtual_daa_score, prm, args, results, storage_mass, entries_out, scripts_out, scripts_cap, scripts_used, &iso);
}

// the mempool's admission path (validate_and_insert_transaction.rs:20-33, 142-159) with its standardness policy around the pipeline above
extern "C" int kgv_validate_mempool_txs_with_policy(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, uint64_t virtual_daa_score,
                                                    uint64_t virtual_past_median_time, const kgv_params* prm, const kgv_tx_rules* rules,
                                                    const kgv_mempool_tx_args* args, kgv_tx_result* results, uint64_t* storage_mass, kgv_tx_masses* masses,
                                                    kgv_utxo_entry* entries_out, uint8_t* scripts_out, size_t scripts_cap, size_t* scripts_used,
                                                    const kgv_mempool_policy* policy, uint64_t* detail) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  const MempoolIso iso{rules, virtual_past_median_time, masses, policy, detail};
  return mempool_core(ctx, t, batch, virtual_daa_score, prm, args, results, storage_mass, entries_out, scripts_out, scripts_cap, scripts_used, &iso);
}

extern "C" int kgv_utxo_apply_accepted(kgv_ctx* ctx, kgv_utxo_table* t, const kgv_tx_batch* batch, const uint8_t* accept, uint64_t pov_daa_score) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || (batch->n_txs && !accept)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (batch->n_txs == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_apply_accepted", t, t)) return rc;
  int rc = utxo_reserve(ctx, t, batch->n_outputs + (t->base ? batch->n_inputs : 0), batch->n_bytes + 8 * (uint64_t)batch->n_outputs);
  if (rc) return rc;
  kgv_dev_batch d;
  rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  size_t nt = d.n_txs, ni = d.n_inputs, no = d.n_outputs;
  uint32_t *itx, *otx;
  uint64_t* ids;
  rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap,
                          [&](kgv_carve& c) { itx = c.take<uint32_t>(ni); otx = c.take<uint32_t>(no); ids = c.take<uint64_t>(nt * 4); });
  if (rc) return rc;
  kgv_io io(ctx);
  const uint8_t* dacc;
  io.in(accept, nt, &dacc);
  if ((rc = io.stage())) return rc;
  BatchView v{d.txs, d.inputs, d.outputs, nullptr, d.bytes};
  cudaStream_t st = ctx->stream;
  if ((rc = kgv_tx_digests_run(ctx, d, nt, ids, false))) return rc;
  k_input_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, itx);
  CK(cudaGetLastError());
  k_output_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, otx);
  CK(cudaGetLastError());
  ctx->launches += 2;
  if (ni) { k_apply_erase<<<nblk(ni, 128), 128, 0, st>>>(view_of(t), d.txs, d.inputs, ni, itx, dacc); CK(cudaGetLastError()); ctx->launches++; }
  if (no) { k_apply_insert<<<nblk(no, 128), 128, 0, st>>>(view_of(t), v, no, otx, dacc, ids, pov_daa_score); CK(cudaGetLastError()); ctx->launches++; }
  if (!io.is_device(accept)) CK(cudaStreamSynchronize(st));  // a host-pointer call returns with the table updated
  return KGV_OK;
}

// ---------------------------------------------------------------------------------------------
// K8 entry points
// ---------------------------------------------------------------------------------------------
extern "C" int kgv_muhash_txs(kgv_ctx* ctx, kgv_utxo_table* table, const kgv_tx_batch* batch, const uint8_t* accept, uint64_t pov_daa_score,
                              uint8_t* numerator384, uint8_t* denominator384) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || !numerator384 || !denominator384 || (batch->n_txs && !accept)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_muhash_txs", {numerator384, denominator384})) return rc;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (table)
    if (int rc = acc.acquire("kgv_muhash_txs", table)) return rc;
  kgv_dev_batch d;
  d.n_txs = d.n_inputs = d.n_outputs = d.n_bytes = 0;
  if (batch->n_txs) {
    int rc = kgv_batch_to_device(ctx, batch, &d, table == nullptr);
    if (rc) return rc;
  }
  const size_t nt = d.n_txs, ni = d.n_inputs, no = d.n_outputs;
  uint32_t *e_den = nullptr, *e_num = nullptr;
  int rc = kgv_mu_reserve(ctx, ni, no, &e_den, &e_num);
  if (rc) return rc;
  if (nt) {
    DevEntry* dent;
    uint32_t *itx, *otx;
    uint64_t* ids;
    rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap, [&](kgv_carve& c) {
      dent = c.take<DevEntry>(ni); itx = c.take<uint32_t>(ni); otx = c.take<uint32_t>(no); ids = c.take<uint64_t>(nt * 4);
    });
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    const uint8_t* dacc;
    io.in(accept, nt, &dacc);
    if ((rc = io.stage())) return rc;
    if (ni) {
      if (table) k_populate<<<nblk(ni, 128), 128, 0, st>>>(view_of(table), d.inputs, ni, dent);
      else k_entries_from_batch<<<nblk(ni, 128), 128, 0, st>>>(d.entries, d.bytes, ni, dent);
      CK(cudaGetLastError());
      ctx->launches++;
    }
    BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
    if ((rc = kgv_tx_digests_run(ctx, d, nt, ids, false))) return rc;
    k_input_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, itx);
    CK(cudaGetLastError());
    k_output_tx_index<<<nblk(nt, 128), 128, 0, st>>>(d.txs, (uint32_t)nt, otx);
    CK(cudaGetLastError());
    if (ni + no) {
      k_muhash_tx_elements<<<nblk(ni + no, 128), 128, 0, st>>>(v, ni, no, itx, otx, dacc, ids, pov_daa_score, e_den, e_num);
      CK(cudaGetLastError());
    }
    ctx->launches += 3;
  }
  return kgv_mu_reduce(ctx, io, ni, no, numerator384, denominator384);
}

// MuHash of the whole UTXO set (the pruning-point / virtual UTXO commitment: MuHash::add_utxo for every entry,
// consensus/core/src/muhash.rs:28-33).  The table is walked in chunks; chunk products are multiplied in a last tree.
extern "C" int kgv_utxo_muhash(kgv_ctx* ctx, kgv_utxo_table* t, uint8_t* numerator384) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!numerator384) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (t->base) { ctx->err = "count / digest / MuHash are defined on plain tables: commit the view first"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_muhash", t)) return rc;
  const uint64_t slots = t->mask + 1;
  const size_t chunk = slots < ((uint64_t)1 << 17) ? (size_t)slots : ((size_t)1 << 17);
  const size_t n_chunks = (size_t)((slots + chunk - 1) / chunk);
  int rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, (n_chunks + 1) * 384);
  if (rc) return rc;
  uint8_t* prods = ctx->d_out;                    // n_chunks x 384 B, contiguous values
  uint8_t* dummy_den = ctx->d_out + n_chunks * 384;
  kgv_io io(ctx);
  for (size_t c = 0; c < n_chunks; c++) {
    const uint64_t first = (uint64_t)c * chunk;
    const size_t n = (size_t)((slots - first) < chunk ? (slots - first) : chunk);
    uint32_t *e_den = nullptr, *e_num = nullptr;
    rc = kgv_mu_reserve(ctx, 0, n, &e_den, &e_num);
    if (rc) return rc;
    k_muhash_table_elements<<<nblk(n, 128), 128, 0, ctx->stream>>>(view_of(t), first, n, e_num);
    CK(cudaGetLastError());
    ctx->launches++;
    rc = kgv_mu_reduce(ctx, io, 0, n, prods + 384 * c, dummy_den);
    if (rc) return rc;
  }
  if (n_chunks == 1) return (rc = io.copy_out(numerator384, prods, 384)) ? rc : io.finish();
  uint32_t *e_den = nullptr, *e_num = nullptr;
  rc = kgv_mu_reserve(ctx, 0, n_chunks, &e_den, &e_num);
  if (rc) return rc;
  k_u3072_scatter<<<nblk(n_chunks, 128), 128, 0, ctx->stream>>>((const uint32_t*)prods, n_chunks, e_num);
  CK(cudaGetLastError());
  ctx->launches++;
  uint8_t den_host[384];  // the denominator goes to the numerator's side
  return kgv_mu_reduce(ctx, io, 0, n_chunks, numerator384, io.is_device(numerator384) ? dummy_den : den_host);
}

#include "kgv_replay_impl.cuh"
