// kgv_hash.cu — tx id / tx hash / sighash kernels and their C ABI entry points (include/kgv.h).
// One hash per thread; the tx records are read once, the digests written once: these kernels stream
// the batch (HBM-bound side of the path, SURVEY.md §8d) — the ALU work is 12 BLAKE2b rounds per 128 B.
#include "kgv_internal.h"
#include "kgv_txhash.cuh"
#include "kgv_muhash.cuh"

#include <cstdio>
#include <string>

using namespace kgv;


// range checks of a HOST batch (a device-resident batch is trusted: its producer is device code of the same process)
static int kgv_check_host_batch(std::string& err_out, const kgv_tx_batch* b) {
  struct { std::string& err; } ctx_{err_out};
  auto* ctx = &ctx_;
  // the records are about to drive device-side pointer arithmetic, so every range is checked first
  for (size_t i = 0; i < b->n_txs; i++) {
    const kgv_tx& t = b->txs[i];
    if ((uint64_t)t.first_input + t.n_inputs > b->n_inputs || (uint64_t)t.first_output + t.n_outputs > b->n_outputs ||
        (uint64_t)t.payload_off + t.payload_len > b->n_bytes) {
      ctx->err = "malformed batch: transaction " + std::to_string(i) + " points outside the input / output / byte arrays";
      return KGV_ERR_ARG;
    }
  }
  // the per-transaction ranges must tile inputs[] and outputs[] exactly, in order: the kernels derive the input -> transaction and
  // output -> transaction maps from them (an input no range covers would index verdict arrays with an uninitialised number)
  {
    uint64_t at_in = 0, at_out = 0;
    for (size_t i = 0; i < b->n_txs; i++) {
      const kgv_tx& t = b->txs[i];
      if (t.first_input != at_in || t.first_output != at_out) {
        ctx->err = "malformed batch: transaction " + std::to_string(i) + " does not continue the input / output ranges of its predecessor";
        return KGV_ERR_ARG;
      }
      at_in += t.n_inputs; at_out += t.n_outputs;
    }
    if (at_in != b->n_inputs || at_out != b->n_outputs) { ctx->err = "malformed batch: the transactions do not cover the input / output arrays"; return KGV_ERR_ARG; }
  }
  for (size_t i = 0; i < b->n_inputs; i++)
    if ((uint64_t)b->inputs[i].sigscript_off + b->inputs[i].sigscript_len > b->n_bytes) {
      ctx->err = "malformed batch: signature script of input " + std::to_string(i) + " lies outside the byte arena";
      return KGV_ERR_ARG;
    }
  for (size_t i = 0; i < b->n_outputs; i++)
    if ((uint64_t)b->outputs[i].script_off + b->outputs[i].script_len > b->n_bytes) {
      ctx->err = "malformed batch: script of output " + std::to_string(i) + " lies outside the byte arena";
      return KGV_ERR_ARG;
    }
  if (b->entries)
    for (size_t i = 0; i < b->n_inputs; i++)
      if (!b->entries[i].pad_[0] && (uint64_t)b->entries[i].script_off + b->entries[i].script_len > b->n_bytes) {
        ctx->err = "malformed batch: script of entry " + std::to_string(i) + " lies outside the byte arena";
        return KGV_ERR_ARG;
      }
  return KGV_OK;
}
struct BatchLayout { size_t o_tx, o_in, o_out, o_ent, o_by, total; };
static BatchLayout kgv_batch_layout(const kgv_tx_batch* b) {
  BatchLayout L;
  L.o_tx = 0;
  L.o_in = al256(L.o_tx + b->n_txs * sizeof(kgv_tx));
  L.o_out = al256(L.o_in + b->n_inputs * sizeof(kgv_input));
  L.o_ent = al256(L.o_out + b->n_outputs * sizeof(kgv_output));
  L.o_by = al256(L.o_ent + (b->entries ? b->n_inputs * sizeof(kgv_utxo_entry) : 0));
  L.total = al256(L.o_by + b->n_bytes + 16);
  return L;
}
static int kgv_batch_upload(kgv_ctx* ctx, const kgv_tx_batch* b, uint8_t* d, const BatchLayout& L, cudaStream_t st) {
  if (b->n_txs) CK(cudaMemcpyAsync(d + L.o_tx, b->txs, b->n_txs * sizeof(kgv_tx), cudaMemcpyHostToDevice, st));
  if (b->n_inputs) CK(cudaMemcpyAsync(d + L.o_in, b->inputs, b->n_inputs * sizeof(kgv_input), cudaMemcpyHostToDevice, st));
  if (b->n_outputs) CK(cudaMemcpyAsync(d + L.o_out, b->outputs, b->n_outputs * sizeof(kgv_output), cudaMemcpyHostToDevice, st));
  if (b->entries && b->n_inputs) CK(cudaMemcpyAsync(d + L.o_ent, b->entries, b->n_inputs * sizeof(kgv_utxo_entry), cudaMemcpyHostToDevice, st));
  if (b->n_bytes) CK(cudaMemcpyAsync(d + L.o_by, b->bytes, b->n_bytes, cudaMemcpyHostToDevice, st));
  return KGV_OK;
}
static void kgv_batch_pointers(kgv_dev_batch* out, const kgv_tx_batch* b, uint8_t* d, const BatchLayout& L) {
  out->txs = (const kgv_tx*)(d + L.o_tx);
  out->inputs = (const kgv_input*)(d + L.o_in);
  out->outputs = (const kgv_output*)(d + L.o_out);
  out->entries = b->entries ? (const kgv_utxo_entry*)(d + L.o_ent) : nullptr;
  out->bytes = d + L.o_by;
}

// Upload of a host batch AHEAD of its use: checked here, copied on a side stream into one of two prefetch buffers; the call that is later handed
// exactly this batch (same arrays, same sizes) computes straight out of that buffer instead of uploading.  The arrays must stay unchanged
// (and page-locked, for the copy to be asynchronous) until that call.  Typical use: prefetch(window i+1), then the synchronous call for window i.
extern "C" int kgv_batch_prefetch(kgv_ctx* ctx, const kgv_tx_batch* b) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!b) { ctx->err = "null batch"; return KGV_ERR_ARG; }
  if ((b->n_txs && !b->txs) || (b->n_inputs && !b->inputs) || (b->n_outputs && !b->outputs) || (b->n_bytes && !b->bytes)) { ctx->err = "batch array missing"; return KGV_ERR_ARG; }
  const void* probe = b->n_txs ? (const void*)b->txs : (const void*)b->bytes;
  if (!probe || kgv_ptr_is_device(probe)) return KGV_OK;  // nothing to upload
  CK(cudaSetDevice(ctx->device));
  int k = !ctx->prefetch[0].valid ? 0 : (!ctx->prefetch[1].valid ? 1 : ctx->prefetch_next);
  ctx->prefetch_next = k ^ 1;
  auto& P = ctx->prefetch[k];
  if (P.worker.joinable()) P.worker.join();
  P.valid = false;
  if (ctx->last_replay.valid && P.buf && (const uint8_t*)ctx->last_replay.txs >= P.buf && (const uint8_t*)ctx->last_replay.txs < P.buf + P.cap)
    ctx->last_replay.valid = false;  // the window kgv_replay_muhash would read lives in this slot: it has to be asked for before the slot is reused
  const BatchLayout L = kgv_batch_layout(b);
  int rc = kgv_reserve(ctx, &P.buf, &P.cap, L.total);
  if (rc) return rc;
  if (!P.done) CK(cudaEventCreateWithFlags(&P.done, cudaEventDisableTiming));
  if (!ctx->ev_prefetch) CK(cudaEventCreateWithFlags(&ctx->ev_prefetch, cudaEventDisableTiming));
  if (!ctx->copy_stream) CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  // the slot may have fed an earlier call: everything enqueued so far has to be done with it before it is overwritten
  CK(cudaEventRecord(ctx->ev_prefetch, ctx->stream));
  CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_prefetch, 0));
  P.txs = b->txs; P.inputs = b->inputs; P.outputs = b->outputs; P.entries = b->entries; P.bytes = b->bytes;
  P.n_txs = b->n_txs; P.n_inputs = b->n_inputs; P.n_outputs = b->n_outputs; P.n_bytes = b->n_bytes;
  P.rc = KGV_OK;
  P.err.clear();
  // The range checks stream over every record of the batch (~3 ms for a 150 k-transaction window): they and the copy calls run on a worker
  // thread, so that the caller can issue the current window's call right away.  The worker touches only this slot, the copy stream and the
  // caller's (unchanging) arrays; whoever consumes or reuses the slot joins it first.
  const kgv_tx_batch copy = *b;
  const int device = ctx->device;
  cudaStream_t cs = ctx->copy_stream;
  kgv_ctx::PrefetchSlot* slot = &P;
  P.worker = std::thread([copy, device, cs, slot, L]() {
    slot->rc = kgv_check_host_batch(slot->err, &copy);
    if (slot->rc) return;
    cudaError_t e = cudaSetDevice(device);
    uint8_t* d = slot->buf;
    auto cp = [&](size_t off, const void* src, size_t bytes) { if (e == cudaSuccess && bytes) e = cudaMemcpyAsync(d + off, src, bytes, cudaMemcpyHostToDevice, cs); };
    cp(L.o_tx, copy.txs, copy.n_txs * sizeof(kgv_tx));
    cp(L.o_in, copy.inputs, copy.n_inputs * sizeof(kgv_input));
    cp(L.o_out, copy.outputs, copy.n_outputs * sizeof(kgv_output));
    if (copy.entries) cp(L.o_ent, copy.entries, copy.n_inputs * sizeof(kgv_utxo_entry));
    cp(L.o_by, copy.bytes, copy.n_bytes);
    if (e == cudaSuccess) e = cudaEventRecord(slot->done, cs);
    if (e != cudaSuccess) { slot->rc = KGV_ERR_CUDA; slot->err = std::string("kgv_batch_prefetch: ") + cudaGetErrorString(e); }
  });
  P.valid = true;
  return KGV_OK;
}

int kgv_batch_to_device(kgv_ctx* ctx, const kgv_tx_batch* b, kgv_dev_batch* out, bool need_entries) {
  if (!b) { ctx->err = "null batch"; return KGV_ERR_ARG; }
  ctx->last_replay.valid = false;  // whatever the last replay staged may be overwritten from here on
  if ((b->n_txs && !b->txs) || (b->n_inputs && !b->inputs) || (b->n_outputs && !b->outputs) || (b->n_bytes && !b->bytes) ||
      (need_entries && b->n_inputs && !b->entries)) {
    ctx->err = "batch array missing";
    return KGV_ERR_ARG;
  }
  bool dev;
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_tx_batch", {b->txs, b->inputs, b->outputs, b->entries, b->bytes}, &dev)) return rc;
  out->n_txs = b->n_txs; out->n_inputs = b->n_inputs; out->n_outputs = b->n_outputs; out->n_bytes = b->n_bytes;
  if (dev) {
    out->txs = b->txs; out->inputs = b->inputs; out->outputs = b->outputs; out->entries = b->entries; out->bytes = b->bytes;
    return KGV_OK;
  }
  for (auto& P : ctx->prefetch)
    if (P.valid && P.txs == b->txs && P.inputs == b->inputs && P.outputs == b->outputs && P.entries == b->entries && P.bytes == b->bytes && P.n_txs == b->n_txs &&
        P.n_inputs == b->n_inputs && P.n_outputs == b->n_outputs && P.n_bytes == b->n_bytes && (!need_entries || b->entries)) {
      // this very batch was uploaded ahead of time (kgv_batch_prefetch): compute out of its buffer
      P.valid = false;
      if (P.worker.joinable()) P.worker.join();
      if (P.rc) { ctx->err = P.err; return P.rc; }
      CK(cudaStreamWaitEvent(ctx->stream, P.done, 0));
      kgv_batch_pointers(out, b, P.buf, kgv_batch_layout(b));
      return KGV_OK;
    }
  {
    int rc0 = kgv_check_host_batch(ctx->err, b);
    if (rc0) return rc0;
  }
  const BatchLayout L = kgv_batch_layout(b);
  int rc = kgv_reserve(ctx, &ctx->d_batch, &ctx->d_batch_cap, L.total);
  if (rc) return rc;
  rc = kgv_batch_upload(ctx, b, ctx->d_batch, L, ctx->stream);
  if (rc) return rc;
  kgv_batch_pointers(out, b, ctx->d_batch, L);
  return KGV_OK;
}

// ---------------------------------------------------------------------------------------------
template <bool HASH>
__global__ void __launch_bounds__(128) k_tx_digest(BatchView b, uint32_t n_txs, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_txs) return;
  uint64_t d[4];
  if (HASH) tx_hash(d, b, i); else tx_id(d, b, i);
#pragma unroll
  for (int k = 0; k < 4; k++) out[4 * (size_t)i + k] = d[k];
}

__global__ void __launch_bounds__(128) k_sighash_reused(BatchView b, uint32_t n_txs, SigHashReused* __restrict__ reused) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_txs) return;
  SigHashReused r;
  sighash_reused(r, b, i);
  reused[i] = r;
}

__global__ void k_entries_to_dev(const kgv_utxo_entry* __restrict__ in, const uint8_t* __restrict__ bytes, size_t n, DevEntry* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  kgv_utxo_entry e = in[i];
  DevEntry d;
  d.amount = e.amount; d.block_daa_score = e.block_daa_score; d.script = bytes + e.script_off; d.script_len = e.script_len;
  d.spk_version = e.spk_version; d.is_coinbase = e.is_coinbase; d.found = 1;
  out[i] = d;
}

__global__ void __launch_bounds__(128)
k_sighash_items(BatchView b, const SigHashReused* __restrict__ reused, const kgv_sighash_item* __restrict__ items, size_t n_items,
                uint32_t n_txs, uint32_t n_inputs, uint32_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_items) return;
  kgv_sighash_item it = items[i];
  uint32_t w[8];
  if (it.tx >= n_txs || it.input >= n_inputs || !sighash_type_allowed(it.hash_type)) {
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = 0xFFFFFFFFu;
  } else {
    SigHashReused r = reused[it.tx];
    sighash_final(w, b, it.tx, it.input, it.hash_type, it.ecdsa != 0, r);
  }
#pragma unroll
  for (int k = 0; k < 8; k++) out[8 * i + k] = bswap32(w[k]);  // back to the digest's byte order
}

int kgv_tx_digests_run(kgv_ctx* ctx, const kgv_dev_batch& d, size_t n, uint64_t* out, bool hash) {
  if (n == 0) return KGV_OK;
  const BatchView v{d.txs, d.inputs, d.outputs, nullptr, d.bytes};
  const unsigned blocks = (unsigned)((n + 127) / 128);
  if (hash) k_tx_digest<true><<<blocks, 128, 0, ctx->stream>>>(v, (uint32_t)n, out);
  else k_tx_digest<false><<<blocks, 128, 0, ctx->stream>>>(v, (uint32_t)n, out);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

// ---------------------------------------------------------------------------------------------
static int digest_common(kgv_ctx* ctx, const kgv_tx_batch* batch, uint8_t* out32, bool hash) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || (batch->n_txs && !out32)) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (batch->n_txs == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, false);
  if (rc) return rc;
  kgv_io io(ctx);
  uint8_t* dout;
  io.out(out32, d.n_txs * 32, &dout);
  if ((rc = io.stage())) return rc;
  if ((rc = kgv_tx_digests_run(ctx, d, d.n_txs, (uint64_t*)dout, hash))) return rc;
  return io.finish();
}
extern "C" int kgv_tx_ids(kgv_ctx* ctx, const kgv_tx_batch* batch, uint8_t* out32) { return digest_common(ctx, batch, out32, false); }
extern "C" int kgv_tx_hashes(kgv_ctx* ctx, const kgv_tx_batch* batch, uint8_t* out32) { return digest_common(ctx, batch, out32, true); }

extern "C" int kgv_sighash(kgv_ctx* ctx, const kgv_tx_batch* batch, const kgv_sighash_item* items, size_t n_items, uint8_t* out32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!batch || (n_items && (!items || !out32))) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (n_items == 0) return KGV_OK;
  CK(cudaSetDevice(ctx->device));
  kgv_dev_batch d;
  int rc = kgv_batch_to_device(ctx, batch, &d, true);
  if (rc) return rc;
  kgv_io io(ctx);
  if ((rc = io.one_side("kgv_sighash", {items, out32}))) return rc;
  SigHashReused* dre;
  DevEntry* dent;
  rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap,
                          [&](kgv_carve& c) { dre = c.take<SigHashReused>(d.n_txs); dent = c.take<DevEntry>(d.n_inputs, 256); });
  if (rc) return rc;
  const kgv_sighash_item* ditems;
  uint8_t* dout;
  io.in(items, n_items * sizeof(kgv_sighash_item), &ditems);
  io.out(out32, n_items * 32, &dout);
  if ((rc = io.stage())) return rc;
  if (d.n_inputs) {
    k_entries_to_dev<<<(unsigned)((d.n_inputs + 127) / 128), 128, 0, ctx->stream>>>(d.entries, d.bytes, d.n_inputs, dent);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  BatchView v{d.txs, d.inputs, d.outputs, dent, d.bytes};
  k_sighash_reused<<<(unsigned)((d.n_txs + 127) / 128), 128, 0, ctx->stream>>>(v, (uint32_t)d.n_txs, dre);
  CK(cudaGetLastError());
  k_sighash_items<<<(unsigned)((n_items + 127) / 128), 128, 0, ctx->stream>>>(v, dre, ditems, n_items, (uint32_t)d.n_txs, (uint32_t)d.n_inputs, (uint32_t*)dout);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return io.finish();
}

// ---------------------------------------------------------------------------------------------
// Merkle roots (crypto/merkle/src/lib.rs:3-30): many independent trees (one per block) level by level; one thread per
// pair.  Group g owns positions [first[g], first[g+1]) of the flattened hash array; after `level` levels it has
// have = ceil(n_g / 2^level) nodes left, packed at the start of its range.  A finished group (have == 1) carries its
// root forward so that every root ends in the same buffer.
// ---------------------------------------------------------------------------------------------
__global__ void k_merkle_group_index(const uint32_t* __restrict__ first, uint32_t n_groups, uint32_t* __restrict__ gid) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  for (uint32_t p = first[g]; p < first[g + 1]; p++) gid[p] = g;
}
__global__ void __launch_bounds__(128) k_merkle_level(const uint64_t* __restrict__ cur, uint64_t* __restrict__ nxt, const uint32_t* __restrict__ first,
                                                      uint32_t n_groups, const uint32_t* __restrict__ gid, size_t n_cap, uint32_t level) {
  size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_cap || p >= first[n_groups]) return;
  const uint32_t g = gid[p];
  const uint32_t f = first[g], n = first[g + 1] - f;
  const uint32_t li = (uint32_t)(p - f);
  const uint32_t have = (uint32_t)((((uint64_t)n) + ((1ull << level) - 1)) >> level);
  if (have == 1) {  // finished: carry the root
    if (li == 0) {
#pragma unroll
      for (int k = 0; k < 4; k++) nxt[4 * (size_t)f + k] = cur[4 * (size_t)f + k];
    }
    return;
  }
  const uint32_t nh = (have + 1) / 2;
  if (li >= nh) return;
  Blake2b h;
  b2b_init_keyed_words(h, 0x7242656C6B72654Dull, 0x6873614868636E61ull, 16);  // "MerkleBranchHash"
#pragma unroll
  for (int k = 0; k < 4; k++) b2b_u64(h, cur[4 * ((size_t)f + 2 * li) + k]);
  const bool right = 2 * li + 1 < have;
#pragma unroll
  for (int k = 0; k < 4; k++) b2b_u64(h, right ? cur[4 * ((size_t)f + 2 * li + 1) + k] : 0ull);  // missing right child: ZERO_HASH
  uint64_t d[4];
  b2b_final(h, d);
#pragma unroll
  for (int k = 0; k < 4; k++) nxt[4 * ((size_t)f + li) + k] = d[k];
}
__global__ void k_merkle_collect(const uint64_t* __restrict__ cur, const uint32_t* __restrict__ first, uint32_t n_groups, uint64_t* __restrict__ roots) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const bool empty = first[g + 1] == first[g];
#pragma unroll
  for (int k = 0; k < 4; k++) roots[4 * (size_t)g + k] = empty ? 0ull : cur[4 * (size_t)first[g] + k];  // no hashes: ZERO_HASH
}

// dh: device array of up to n_cap hashes (modified: used as one of the two ping-pong buffers); dfirst: n_groups + 1 DEVICE offsets
void kgv_merkle_work::carve(kgv_carve& c, size_t n_cap) { gid = c.take<uint32_t>(n_cap); other = c.take<uint64_t>(n_cap * 4, 32); }
int kgv_merkle_levels(kgv_ctx* ctx, uint64_t* dh, size_t n_cap, const uint32_t* dfirst, uint32_t n_groups, uint32_t max_n, const kgv_merkle_work& w,
                      uint64_t* droots, cudaStream_t st) {
  if (n_cap) {
    k_merkle_group_index<<<(n_groups + 127) / 128, 128, 0, st>>>(dfirst, n_groups, w.gid);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  uint64_t* cur = dh;
  uint64_t* nxt = w.other;
  for (uint32_t level = 0; ((uint64_t)1 << level) < max_n; level++) {
    k_merkle_level<<<(unsigned)((n_cap + 127) / 128), 128, 0, st>>>(cur, nxt, dfirst, n_groups, w.gid, n_cap, level);
    CK(cudaGetLastError());
    ctx->launches++;
    uint64_t* t = cur; cur = nxt; nxt = t;
  }
  k_merkle_collect<<<(n_groups + 127) / 128, 128, 0, st>>>(cur, dfirst, n_groups, droots);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

// first_host: n_groups + 1 offsets on the HOST, from 0 to n_total
int kgv_merkle_run(kgv_ctx* ctx, uint64_t* dh, size_t n_total, const uint32_t* first_host, uint32_t n_groups, uint64_t* droots) {
  uint32_t max_n = 0;
  if (n_groups && (first_host[0] != 0 || first_host[n_groups] != n_total)) { ctx->err = "merkle group offsets must start at 0 and end at the number of hashes"; return KGV_ERR_ARG; }
  for (uint32_t g = 0; g < n_groups; g++) {
    if (first_host[g + 1] < first_host[g] || first_host[g + 1] > n_total) { ctx->err = "merkle group offsets not monotone / out of range"; return KGV_ERR_ARG; }
    uint32_t n = first_host[g + 1] - first_host[g];
    if (n > max_n) max_n = n;
  }
  uint32_t* dfirst;
  kgv_merkle_work w;
  int rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap, [&](kgv_carve& c) { dfirst = c.take<uint32_t>(n_groups + 1); w.carve(c, n_total); });
  if (rc) return rc;
  CK(cudaMemcpyAsync(dfirst, first_host, (n_groups + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
  return kgv_merkle_levels(ctx, dh, n_total, dfirst, n_groups, max_n, w, droots, ctx->stream);
}

extern "C" int kgv_merkle_roots(kgv_ctx* ctx, const uint8_t* hashes32, const uint32_t* first, uint32_t n_groups, uint8_t* roots32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n_groups == 0) return KGV_OK;
  if (!first || !roots32) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_merkle_roots", "first", first)) return rc;
  const size_t n_total = first[n_groups];
  if (n_total && !hashes32) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  int rc = io.one_side("kgv_merkle_roots", {n_total ? hashes32 : nullptr, roots32});
  if (rc) return rc;
  // working copy of the hashes (the tree overwrites its input buffer) + device roots
  uint64_t *dh, *dr;
  rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) { dh = c.take<uint64_t>(n_total * 4, 32); dr = c.take<uint64_t>((size_t)n_groups * 4); });
  if (rc) return rc;
  if (n_total) CK(cudaMemcpyAsync(dh, hashes32, n_total * 32, cudaMemcpyDefault, ctx->stream));
  if ((rc = kgv_merkle_run(ctx, dh, n_total, first, n_groups, dr))) return rc;
  if ((rc = io.copy_out(roots32, dr, (size_t)n_groups * 32))) return rc;
  return io.finish();
}

// calc_hash_merkle_root (consensus/core/src/merkle.rs:5-7) for every block of a batch: block b = transactions
// [block_first_tx[b], block_first_tx[b+1]) (host array); tx hashes never leave the device.
extern "C" int kgv_block_hash_merkle_roots(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks, uint8_t* roots32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n_blocks == 0) return KGV_OK;
  if (!batch || !block_first_tx || !roots32) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_block_hash_merkle_roots", "block_first_tx", block_first_tx)) return rc;
  if (block_first_tx[n_blocks] > batch->n_txs) { ctx->err = "block offsets exceed the batch"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_dev_batch d;
  d.n_txs = 0;
  if (batch->n_txs) {
    int rc = kgv_batch_to_device(ctx, batch, &d, false);
    if (rc) return rc;
  }
  const size_t nt = block_first_tx[n_blocks];
  uint64_t *dh, *dr;
  int rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) { dh = c.take<uint64_t>(nt * 4, 32); dr = c.take<uint64_t>((size_t)n_blocks * 4); });
  if (rc) return rc;
  rc = kgv_tx_digests_run(ctx, d, nt, dh, true);
  if (rc) return rc;
  rc = kgv_merkle_run(ctx, dh, nt, block_first_tx, n_blocks, dr);
  if (rc) return rc;
  kgv_io io(ctx);
  if ((rc = io.copy_out(roots32, dr, (size_t)n_blocks * 32))) return rc;
  return io.finish();
}

// ---------------------------------------------------------------------------------------------
// Block-body set checks (consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:95-131), many blocks at
// once: the hashed sets of kgv_block_body.cu find each check's FIRST offender in the reference's iteration order.
// ---------------------------------------------------------------------------------------------
using BlockCheckAcc = kgv_block_check_acc;

__global__ void k_block_set_checks_final(const BlockCheckAcc* __restrict__ acc, uint32_t n_blocks, kgv_block_check* __restrict__ out) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  BlockCheckAcc a = acc[b];
  kgv_block_check r;
  // order of validate_body_in_isolation (:13-23): duplicates, then double spends, then chained transactions
  if (a.dup_tx != 0xFFFFFFFFu) { r.status = KGV_BLOCK_DUPLICATE_TRANSACTIONS; r.index = a.dup_tx; }
  else if (a.double_spend != 0xFFFFFFFFu) { r.status = KGV_BLOCK_DOUBLE_SPEND_IN_SAME_BLOCK; r.index = a.double_spend; }
  else if (a.chained != 0xFFFFFFFFu) { r.status = KGV_BLOCK_CHAINED_TRANSACTION; r.index = a.chained; }
  else { r.status = KGV_BLOCK_OK; r.index = 0; }
  out[b] = r;
}

extern "C" int kgv_block_set_checks(kgv_ctx* ctx, const kgv_tx_batch* batch, const uint32_t* block_first_tx, uint32_t n_blocks, kgv_block_check* out) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n_blocks == 0) return KGV_OK;
  if (!batch || !block_first_tx || !out) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  if (int rc = kgv_host_only(ctx, "kgv_block_set_checks", "block_first_tx", block_first_tx)) return rc;
  if (batch->n_txs > 0x7FFFFFFFull || batch->n_inputs > 0x7FFFFFFFull) { ctx->err = "kgv_block_set_checks: more than 2^31 - 1 transactions or inputs"; return KGV_ERR_ARG; }
  for (uint32_t b = 0; b < n_blocks; b++)
    if (block_first_tx[b + 1] < block_first_tx[b] || block_first_tx[b + 1] > batch->n_txs) { ctx->err = "block offsets not monotone / out of range"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_dev_batch d;
  d.n_txs = d.n_inputs = 0;
  if (batch->n_txs) {
    int rc = kgv_batch_to_device(ctx, batch, &d, false);
    if (rc) return rc;
  }
  const size_t nt = block_first_tx[n_blocks];
  uint64_t* ids;
  uint32_t* first;
  BlockCheckAcc* acc;
  kgv_block_check* dout;
  kgv_body_sets_work sets;
  int rc = kgv_reserve_carved(ctx, &ctx->d_scratch, &ctx->d_scratch_cap, [&](kgv_carve& c) {
    ids = c.take<uint64_t>(nt * 4, 32); first = c.take<uint32_t>(n_blocks + 1); acc = c.take<BlockCheckAcc>(n_blocks); dout = c.take<kgv_block_check>(n_blocks);
    sets.carve(c, nt, d.n_inputs);
  });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  CK(cudaMemcpyAsync(first, block_first_tx, (n_blocks + 1) * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(acc, 0xFF, (size_t)n_blocks * sizeof(BlockCheckAcc), st));
  if (nt) {
    rc = kgv_tx_digests_run(ctx, d, nt, ids, false);
    if (rc) return rc;
    rc = kgv_body_sets_run(ctx, d, nt, ids, first, n_blocks, acc, sets, st);
    if (rc) return rc;
  }
  k_block_set_checks_final<<<(n_blocks + 127) / 128, 128, 0, st>>>(acc, n_blocks, dout);
  CK(cudaGetLastError());
  ctx->launches++;
  kgv_io io(ctx);
  if ((rc = io.copy_out(out, dout, (size_t)n_blocks * sizeof(kgv_block_check)))) return rc;
  return io.finish();
}
