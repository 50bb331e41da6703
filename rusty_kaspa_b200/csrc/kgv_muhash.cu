// kgv_muhash.cu — K8: MuHash product trees and the element-level entry points of include/kgv.h.
//
// Data flow: one thread builds one 3072-bit element (keyed BLAKE2b -> ChaCha20 keystream) straight into the level-0
// array of its tree; each tree level halves the array with one u3072 multiplication per thread (kgv_u3072.cuh) until
// one value is left; the last kernel writes the canonical residue.  The two trees of a MuHash (numerator = added
// elements, denominator = removed elements, crypto/muhash/src/lib.rs:32-35) run on two streams.
// Algorithmic traffic per multiplication: 2 x 384 B read, 384 B written (+ 1.5 KB scratch row written and re-read);
// the work is 9 216 IMAD.WIDE per multiplication: integer-issue bound like the signature kernels.
#include "kgv_internal.h"
#include "kgv_muhash.cuh"

#include <cstdio>

using namespace kgv;


// one level of a product tree: out[t] = in[2t] * in[2t+1] (the odd element out is copied)
__global__ void __launch_bounds__(128) k_u3072_tree_level(const uint32_t* __restrict__ in, size_t n_in, uint32_t* __restrict__ out, uint32_t* __restrict__ wide) {
  const size_t n_out = (n_in + 1) / 2;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_out) return;
  if (2 * t + 1 < n_in) {
    u3072_mul_mod(out, n_out, t, wide, n_out, t, in, n_in, 2 * t, in, n_in, 2 * t + 1);
  } else {
    for (int i = 0; i < KGV_U3072_BLOCKS; i++) {
      uint32_t r[8];
      u3072_load_block(r, in, n_in, 2 * t, i);
      u3072_store_block(out, n_out, t, i, r);
    }
  }
}
// the same level with one multiplication per 16-lane group (kgv_u3072.cuh, cooperative form): ~10x shorter per-level
// latency, used while a level has too few multiplications to fill the machine with one thread each
#define KGV_COOP_GROUPS 8  // groups (multiplications) per 128-thread block
__global__ void __launch_bounds__(128) k_u3072_tree_level_coop(const uint32_t* __restrict__ in, size_t n_in, uint32_t* __restrict__ out) {
  __shared__ U3072Coop sm[KGV_COOP_GROUPS];
  const size_t n_out = (n_in + 1) / 2;
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const size_t t = (size_t)blockIdx.x * KGV_COOP_GROUPS + grp;
  const bool have = t < n_out;
  const bool mul = have && 2 * t + 1 < n_in;
  u3072_coop_mul_mod(sm[grp], lane, mul, out, n_out, t, in, n_in, 2 * t, in, n_in, 2 * t + 1);
  if (have && !mul && lane < KGV_U3072_BLOCKS) {
    uint32_t r[8];
    u3072_load_block(r, in, n_in, 2 * t, lane);
    u3072_store_block(out, n_out, t, lane, r);
  }
}

// canonical residue of a single value (stride `s`, element 0) as 384 little-endian bytes; n == 0: the value one
__global__ void k_u3072_emit(const uint32_t* __restrict__ a, size_t s, int is_empty, uint32_t* __restrict__ out96) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (is_empty) {
    out96[0] = 1;
    for (int i = 1; i < 96; i++) out96[i] = 0;
    return;
  }
  uint32_t r[96];
  u3072_canonical(r, a, s, 0);
  for (int i = 0; i < 96; i++) out96[i] = r[i];
}

// raw elements: element i = data[offsets[i] .. offsets[i+1]); remove[i] != 0 puts it in the denominator tree.
// Both trees have n slots; the slot of the other tree holds the identity.
__global__ void __launch_bounds__(128) k_muhash_raw_elements(const uint8_t* __restrict__ data, const uint64_t* __restrict__ offsets, const uint8_t* __restrict__ remove,
                                                             size_t n, uint32_t* __restrict__ e_den, uint32_t* __restrict__ e_num) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Blake2b h;
  b2b_init_muhash_element(h);
  const uint64_t a = offsets[i], b = offsets[i + 1];
  for (uint64_t k = a; k < b; k++) b2b_byte(h, data[k]);
  uint64_t d[4];
  b2b_final(h, d);
  const bool rem = remove && remove[i];
  muhash_expand_store(rem ? e_den : e_num, n, i, d);
  u3072_store_one(rem ? e_num : e_den, n, i);
}

// ---------------------------------------------------------------------------------------------
// tree driver
// ---------------------------------------------------------------------------------------------
// one product tree of n elements in d_mu: level 0, level 1, the wide-product rows and the result (384 bytes in a 512-byte slot)
struct MuTree {
  size_t n;
  uint32_t *lvl0, *lvl1, *wide, *out;
  void carve(kgv_carve& c) {
    lvl0 = c.take<uint32_t>(n * 96); lvl1 = c.take<uint32_t>((n + 1) / 2 * 96); wide = c.take<uint32_t>((n + 1) / 2 * 192); out = c.take<uint32_t>(128);
  }
};
// the two trees of kgv_mu_reserve / kgv_mu_reduce, the denominator's first
struct MuTrees {
  MuTree den, num;
  void carve(kgv_carve& c) { den.carve(c); num.carve(c); }
};

int kgv_mu_reserve(kgv_ctx* ctx, size_t n_den, size_t n_num, uint32_t** e_den, uint32_t** e_num) {
  MuTrees t{{n_den}, {n_num}};
  int rc = kgv_reserve_carved(ctx, &ctx->d_mu, &ctx->d_mu_cap, [&](kgv_carve& c) { t.carve(c); });
  if (rc) return rc;
  *e_den = t.den.lvl0;
  *e_num = t.num.lvl0;
  return KGV_OK;
}

static int reduce_one(kgv_ctx* ctx, const MuTree& m, cudaStream_t st) {
  const size_t n = m.n;
  uint32_t* cur = m.lvl0;
  uint32_t* nxt = m.lvl1;
  size_t k = n;
  while (k > 1) {
    size_t h = (k + 1) / 2;
    if (h <= 8192) k_u3072_tree_level_coop<<<nblk(h, KGV_COOP_GROUPS), 128, 0, st>>>(cur, k, nxt);
    else k_u3072_tree_level<<<nblk(h, 128), 128, 0, st>>>(cur, k, nxt, m.wide);
    CK(cudaGetLastError());
    ctx->launches++;
    uint32_t* t = cur; cur = nxt; nxt = t;
    k = h;
  }
  k_u3072_emit<<<1, 32, 0, st>>>(cur, 1, n == 0 ? 1 : 0, m.out);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

int kgv_mu_reduce(kgv_ctx* ctx, kgv_io& io, size_t n_den, size_t n_num, uint8_t* out_num384, uint8_t* out_den384) {
  cudaStream_t st = ctx->stream, sx = ctx->aux_stream;
  MuTrees t{{n_den}, {n_num}};
  kgv_carve c{ctx->d_mu};  // the layout kgv_mu_reserve gave d_mu
  t.carve(c);
  CK(cudaEventRecord(ctx->ev_fork, st));
  CK(cudaStreamWaitEvent(sx, ctx->ev_fork, 0));
  int rc = reduce_one(ctx, t.den, st);
  if (rc) return rc;
  rc = reduce_one(ctx, t.num, sx);
  if (rc) return rc;
  CK(cudaEventRecord(ctx->ev_join, sx));
  CK(cudaStreamWaitEvent(st, ctx->ev_join, 0));
  if ((rc = io.copy_out(out_den384, t.den.out, 384))) return rc;
  if ((rc = io.copy_out(out_num384, t.num.out, 384))) return rc;
  return io.finish();
}

// ---------------------------------------------------------------------------------------------
// C ABI: element level
// ---------------------------------------------------------------------------------------------
extern "C" int kgv_muhash_elements(kgv_ctx* ctx, const uint8_t* data, const uint64_t* offsets, const uint8_t* remove, size_t n, uint8_t* numerator384,
                                   uint8_t* denominator384) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!numerator384 || !denominator384 || (n && (!offsets || !data))) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  kgv_io io(ctx);
  int rc = io.one_side("kgv_muhash_elements", {numerator384, denominator384});
  if (rc) return rc;
  // device offsets cannot be read here to size a host copy of the data: then data and remove are device arrays too
  if (n && io.is_device(offsets) && (rc = io.one_side("kgv_muhash_elements", {offsets, data, remove}))) return rc;
  CK(cudaSetDevice(ctx->device));
  uint32_t *e_den = nullptr, *e_num = nullptr;
  if ((rc = kgv_mu_reserve(ctx, n, n, &e_den, &e_num))) return rc;
  if (n) {
    const uint8_t *ddata = data, *drem = remove;
    const uint64_t* doff = offsets;
    if (!io.is_device(offsets)) {  // the data's size is the end of the offsets, readable only in host memory
      io.in(data, offsets[n], &ddata);
      io.in(offsets, (n + 1) * 8, &doff);
      io.in(remove, n, &drem);
      if ((rc = io.stage())) return rc;
    }
    k_muhash_raw_elements<<<nblk(n, 128), 128, 0, ctx->stream>>>(ddata, doff, drem, n, e_den, e_num);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  return kgv_mu_reduce(ctx, io, n, n, numerator384, denominator384);
}

// Test / audit hook: one product-tree level on caller values, by the same two level kernels reduce_one launches
extern "C" int kgv_debug_u3072_level(kgv_ctx* ctx, int coop, const uint8_t* in384, size_t n_in, uint8_t* out384) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!in384 || !out384 || n_in == 0 || n_in > ((size_t)1 << 20) || (coop != 0 && coop != 1)) { ctx->err = "bad u3072 level arguments"; return KGV_ERR_ARG; }
  if (kgv_ptr_is_device(in384) || kgv_ptr_is_device(out384)) { ctx->err = "kgv_debug_u3072_level takes host pointers"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  const size_t h = (n_in + 1) / 2;
  uint8_t *lvl, *out, *wide;
  int rc = kgv_reserve_carved(ctx, &ctx->d_mu, &ctx->d_mu_cap,
                              [&](kgv_carve& c) { lvl = c.take<uint8_t>(n_in * 384); out = c.take<uint8_t>(h * 384); wide = c.take<uint8_t>(h * 768); });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  // contiguous values -> block-transposed level (limb block i of element e at (i * n_in + e) * 32 bytes) and back
  for (int i = 0; i < KGV_U3072_BLOCKS; i++)
    CK(cudaMemcpy2DAsync(lvl + (size_t)i * n_in * 32, 32, in384 + 32 * i, 384, 32, n_in, cudaMemcpyHostToDevice, st));
  if (coop) k_u3072_tree_level_coop<<<nblk(h, KGV_COOP_GROUPS), 128, 0, st>>>((const uint32_t*)lvl, n_in, (uint32_t*)out);
  else k_u3072_tree_level<<<nblk(h, 128), 128, 0, st>>>((const uint32_t*)lvl, n_in, (uint32_t*)out, (uint32_t*)wide);
  CK(cudaGetLastError());
  ctx->launches++;
  for (int i = 0; i < KGV_U3072_BLOCKS; i++)
    CK(cudaMemcpy2DAsync(out384 + 32 * i, 384, out + (size_t)i * h * 32, 32, 32, h, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return KGV_OK;
}

// a <- a * b for both fields (crypto/muhash/src/lib.rs:91-96 combine); all four are 384-byte little-endian residues
__global__ void k_muhash_combine(uint32_t* __restrict__ w) {  // w: [a_num | a_den | b_num | b_den] contiguous words; one warp: group 0 numerators, group 1 denominators
  __shared__ U3072Coop sm[2];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  uint32_t* a = w + 96 * grp;
  const uint32_t* b = w + 96 * (2 + grp);
  u3072_coop_mul_mod(sm[grp], lane, true, a, 1, 0, a, 1, 0, b, 1, 0);
  if (lane == 0) {
    uint32_t r[96];
    u3072_canonical(r, a, 1, 0);
    for (int i = 0; i < 96; i++) a[i] = r[i];
  }
}
extern "C" int kgv_muhash_combine(kgv_ctx* ctx, uint8_t* num_a, uint8_t* den_a, const uint8_t* num_b, const uint8_t* den_b) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!num_a || !den_a || !num_b || !den_b) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  int rc = kgv_reserve(ctx, &ctx->d_mu, &ctx->d_mu_cap, 4096);
  if (rc) return rc;
  uint8_t* w = ctx->d_mu;
  kgv_io io(ctx);
  const uint8_t* ins[4] = {num_a, den_a, num_b, den_b};  // each copied in from its own side
  for (int i = 0; i < 4; i++)
    CK(cudaMemcpyAsync(w + 384 * i, ins[i], 384, io.is_device(ins[i]) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
  k_muhash_combine<<<1, 32, 0, ctx->stream>>>((uint32_t*)w);
  CK(cudaGetLastError());
  ctx->launches++;
  if ((rc = io.copy_out(num_a, w, 384)) || (rc = io.copy_out(den_a, w + 384, 384))) return rc;
  return io.finish();
}

// finalize (lib.rs:98-115): serialized = numerator / denominator mod p (canonical), hash = BLAKE2b-256 keyed "MuHashFinalize".
// The inverse is denominator^(p-2): p - 2 = (2^3051 - 1) * 2^21 + 993433, i.e. 3 072 squarings and ~30 multiplications,
// strictly sequential.  OFF the data-parallel path (the reference finalizes once per chain block in sequential code):
// one 16-lane group multiplying cooperatively, a few ms.  w: [num | den | cur | saved] contiguous words; out: 96 words serialized + 8 words hash.
// one real function for the many call sites of the exponentiation ladder (contiguous operands, stride 1)
static __device__ __noinline__ void coop_mul_contig(U3072Coop* sm, int lane, bool act, uint32_t* r, const uint32_t* a, const uint32_t* b) {
  u3072_coop_mul_mod(*sm, lane, act, r, 1, 0, a, 1, 0, b, 1, 0);
}
__global__ void k_muhash_finalize(uint32_t* __restrict__ w, uint32_t* __restrict__ out) {
  __shared__ U3072Coop sm;
  const int lane = threadIdx.x & 15;
  const bool act = threadIdx.x < 16;  // one 16-lane group does the arithmetic; the other half of the warp only keeps the warp syncs company
  uint32_t *num = w, *den = w + 96, *cur = w + 192, *saved = w + 288;
  auto mul = [&](uint32_t* r, const uint32_t* a, const uint32_t* b) { coop_mul_contig(&sm, lane, act, r, a, b); };
  auto copy = [&](uint32_t* d, const uint32_t* s_) {
    if (act) for (int i = lane; i < 96; i += 16) d[i] = s_[i];
    __syncwarp();
  };
  // cur = den^(2^k - 1) with k following the bits of 3051 = 0b101111101011 from the top
  copy(cur, den);
  int k = 1;
  for (int bit = 10; bit >= 0; bit--) {
    copy(saved, cur);
    for (int q = 0; q < k; q++) mul(cur, cur, cur);
    mul(cur, cur, saved);
    k *= 2;
    if ((3051 >> bit) & 1) { mul(cur, cur, cur); mul(cur, cur, den); k += 1; }
  }
  for (int bit = 20; bit >= 0; bit--) {
    mul(cur, cur, cur);
    if ((993433u >> bit) & 1u) mul(cur, cur, den);
  }
  mul(num, num, cur);
  if (threadIdx.x == 0) {
    uint32_t r[96];
    u3072_canonical(r, num, 1, 0);
    Blake2b h;
    b2b_init_muhash_finalize(h);
    for (int i = 0; i < 96; i++) { out[i] = r[i]; b2b_u32(h, r[i]); }
    uint64_t d[4];
    b2b_final(h, d);
    for (int i = 0; i < 4; i++) { out[96 + 2 * i] = (uint32_t)d[i]; out[96 + 2 * i + 1] = (uint32_t)(d[i] >> 32); }
  }
}
extern "C" int kgv_muhash_finalize(kgv_ctx* ctx, const uint8_t* numerator384, const uint8_t* denominator384, uint8_t* serialized384, uint8_t* hash32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!numerator384 || !denominator384 || !hash32) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  uint8_t *w, *o;
  int rc = kgv_reserve_carved(ctx, &ctx->d_mu, &ctx->d_mu_cap, [&](kgv_carve& c) { w = c.take<uint8_t>(4096); o = c.take<uint8_t>(4096); });
  if (rc) return rc;
  kgv_io io(ctx);
  const uint8_t* ins[2] = {numerator384, denominator384};  // each copied in from its own side
  for (int i = 0; i < 2; i++)
    CK(cudaMemcpyAsync(w + 384 * i, ins[i], 384, io.is_device(ins[i]) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
  k_muhash_finalize<<<1, 32, 0, ctx->stream>>>((uint32_t*)w, (uint32_t*)o);
  CK(cudaGetLastError());
  ctx->launches++;
  if (serialized384 && (rc = io.copy_out(serialized384, o, 384))) return rc;
  if ((rc = io.copy_out(hash32, o + 384, 32))) return rc;
  return io.finish();
}


// ---------------------------------------------------------------------------------------------
// Batched MuHash work for a replay window: segmented products, running (prefix) products and ONE modular inversion for any number
// of finalizations.  All values here are contiguous 96-word little-endian residues ("pitch" words apart); every multiplication is
// done by a 16-lane group (u3072_coop_mul_mod), 8 groups per block.
// Reference: MuHash::combine chain of calculate_utxo_state (utxo_validation.rs:144) and MuHash::finalize per chain block (:188-192,
// crypto/muhash/src/lib.rs:98-115).  The reference pays one 3072-bit inversion per chain block; here n finalizations cost one
// inversion + 5n multiplications (Montgomery's trick with prefix / suffix products built by parallel scans).
// Zero is not handled specially (a MuHash element is 0 or p only if a ChaCha20 stream is all-zero / equals p: probability 2^-3072).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void coop_copy(int lane, bool act, uint32_t* dst, const uint32_t* src) {
  if (act && lane < KGV_U3072_BLOCKS) {
    uint32_t r[8];
    u3072_load_block(r, src, 1, 0, lane);
    u3072_store_block(dst, 1, 0, lane, r);
  }
  __syncwarp();
}
__device__ __forceinline__ void coop_set_one(int lane, bool act, uint32_t* dst) {
  if (act && lane < KGV_U3072_BLOCKS) {
    uint32_t r[8] = {lane == 0 ? 1u : 0u, 0, 0, 0, 0, 0, 0, 0};
    u3072_store_block(dst, 1, 0, lane, r);
  }
  __syncwarp();
}

// out[g] = product of the level-0 elements E[lo[g] .. hi[g]) whose flag is set (flags == nullptr: all); empty product = 1
__global__ void __launch_bounds__(128) k_u3072_range_product(const uint32_t* __restrict__ E, size_t stride, const uint8_t* __restrict__ flags, const uint32_t* __restrict__ flag_index,
                                                             const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, uint32_t n_segs, uint32_t* __restrict__ out,
                                                             size_t out_pitch) {
  __shared__ U3072Coop sm[KGV_COOP_GROUPS];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const uint32_t g = blockIdx.x * KGV_COOP_GROUPS + grp;
  const bool mine = g < n_segs;
  const uint32_t a = mine ? lo[g] : 0, b = mine ? hi[g] : 0;
  // both groups of a warp walk in lockstep: the trip count is the longer of the two ranges
  const uint32_t len = b - a;
  const uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, len, 16);
  const uint32_t trips = len > other ? len : other;
  uint32_t* acc = out + out_pitch * (size_t)(mine ? g : 0);
  bool started = false;
  for (uint32_t it = 0; it < trips; it++) {
    const uint32_t j = a + it;
    const bool have = mine && j < b && (!flags || flags[flag_index ? flag_index[j] : j]);
    if (have && !started && lane < KGV_U3072_BLOCKS) {
      uint32_t r[8];
      u3072_load_block(r, E, stride, j, lane);
      u3072_store_block(acc, 1, 0, lane, r);
    }
    __syncwarp();
    u3072_coop_mul_mod(sm[grp], lane, have && started, acc, 1, 0, acc, 1, 0, E, stride, j);
    started = started || have;
  }
  coop_set_one(lane, mine && !started, acc);
}

// element i of a value array with a pitch (in words); rev walks the array backwards
__device__ __forceinline__ uint32_t* u3072_at(uint32_t* base, size_t pitch, size_t n, size_t i, bool rev) { return base + pitch * (rev ? n - 1 - i : i); }

// blocked inclusive scan (products), three launches: chunks in parallel, then the chunk totals, then the carry-in of every chunk
#define KGV_SCAN_CHUNK 32
__global__ void __launch_bounds__(128) k_u3072_scan_chunks(uint32_t* __restrict__ vals, size_t pitch, size_t n, bool rev) {
  __shared__ U3072Coop sm[KGV_COOP_GROUPS];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const size_t c = (size_t)blockIdx.x * KGV_COOP_GROUPS + grp;
  const size_t first = c * KGV_SCAN_CHUNK;
  for (size_t k = 1; k < KGV_SCAN_CHUNK; k++) {
    const bool act = first + k < n;
    uint32_t* cur = u3072_at(vals, pitch, n, act ? first + k : 0, rev);
    const uint32_t* prev = u3072_at(vals, pitch, n, act ? first + k - 1 : 0, rev);
    u3072_coop_mul_mod(sm[grp], lane, act, cur, 1, 0, cur, 1, 0, prev, 1, 0);
  }
}
// tot[c] = product of chunks 0..c (inclusive), sequentially by one group (n / 32 multiplications)
__global__ void __launch_bounds__(32) k_u3072_scan_totals(uint32_t* __restrict__ vals, size_t pitch, size_t n, bool rev, uint32_t* __restrict__ tot) {
  __shared__ U3072Coop sm;
  const int lane = threadIdx.x & 15;
  const bool act = threadIdx.x < 16;
  const size_t n_chunks = (n + KGV_SCAN_CHUNK - 1) / KGV_SCAN_CHUNK;
  for (size_t c = 0; c < n_chunks; c++) {
    const size_t last = (c + 1) * KGV_SCAN_CHUNK - 1 < n ? (c + 1) * KGV_SCAN_CHUNK - 1 : n - 1;
    const uint32_t* v = u3072_at(vals, pitch, n, last, rev);
    if (c == 0) coop_copy(lane, act, tot, v);
    else u3072_coop_mul_mod(sm, lane, act, tot + 96 * c, 1, 0, tot + 96 * (c - 1), 1, 0, v, 1, 0);
  }
}
__global__ void __launch_bounds__(128) k_u3072_scan_apply(uint32_t* __restrict__ vals, size_t pitch, size_t n, bool rev, const uint32_t* __restrict__ tot) {
  __shared__ U3072Coop sm[KGV_COOP_GROUPS];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const size_t i = (size_t)blockIdx.x * KGV_COOP_GROUPS + grp + KGV_SCAN_CHUNK;  // the first chunk has no carry-in
  const bool act = i < n;
  uint32_t* cur = u3072_at(vals, pitch, n, act ? i : 0, rev);
  u3072_coop_mul_mod(sm[grp], lane, act, cur, 1, 0, cur, 1, 0, tot + 96 * (act ? i / KGV_SCAN_CHUNK - 1 : 0), 1, 0);
}
// vals[0] *= init  (start of a running product)
__global__ void __launch_bounds__(32) k_u3072_mul_first(uint32_t* __restrict__ vals, const uint32_t* __restrict__ init, int n_arrays, size_t array_off) {
  __shared__ U3072Coop sm[2];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const bool act = grp < n_arrays;
  uint32_t* v = vals + array_off * (act ? grp : 0);
  u3072_coop_mul_mod(sm[grp], lane, act, v, 1, 0, v, 1, 0, init + 96 * (act ? grp : 0), 1, 0);
}

// inv = a^(p-2): p - 2 = (2^3051 - 1) * 2^21 + 993433 (3 072 squarings, ~30 multiplications), one 16-lane group.  w: [a | cur | saved]
__device__ __forceinline__ void coop_inverse(U3072Coop* sm, int lane, bool act, uint32_t* a, uint32_t* cur, uint32_t* saved) {
  auto mul = [&](uint32_t* r, const uint32_t* x, const uint32_t* y) { coop_mul_contig(sm, lane, act, r, x, y); };
  coop_copy(lane, act, cur, a);
  int k = 1;
  for (int bit = 10; bit >= 0; bit--) {  // cur = a^(2^k - 1), k following the bits of 3051 = 0b101111101011 from the top
    coop_copy(lane, act, saved, cur);
    for (int q = 0; q < k; q++) mul(cur, cur, cur);
    mul(cur, cur, saved);
    k *= 2;
    if ((3051 >> bit) & 1) { mul(cur, cur, cur); mul(cur, cur, a); k += 1; }
  }
  for (int bit = 20; bit >= 0; bit--) {
    mul(cur, cur, cur);
    if ((993433u >> bit) & 1u) mul(cur, cur, a);
  }
}
__global__ void __launch_bounds__(32) k_u3072_inverse_one(uint32_t* __restrict__ w) {
  __shared__ U3072Coop sm;
  coop_inverse(&sm, threadIdx.x & 15, threadIdx.x < 16, w, w + 96, w + 192);
}
// Montgomery's trick, parallel form: inv_i = I * P[i-1] * S[i+1] with P / S the prefix / suffix products of the denominators and
// I = 1 / P[n-1]; then value_i = num_i * inv_i.  out: n contiguous values
__global__ void __launch_bounds__(128) k_muhash_divide_all(const uint32_t* __restrict__ num, size_t num_pitch, const uint32_t* __restrict__ P, const uint32_t* __restrict__ S,
                                                           const uint32_t* __restrict__ I, size_t n, uint32_t* __restrict__ out) {
  __shared__ U3072Coop sm[KGV_COOP_GROUPS];
  const int grp = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const size_t i = (size_t)blockIdx.x * KGV_COOP_GROUPS + grp;
  const bool act = i < n;
  const size_t k = act ? i : 0;
  uint32_t* o = out + 96 * k;
  coop_copy(lane, act, o, I);
  u3072_coop_mul_mod(sm[grp], lane, act && k > 0, o, 1, 0, o, 1, 0, P + 96 * (k > 0 ? k - 1 : 0), 1, 0);
  u3072_coop_mul_mod(sm[grp], lane, act && k + 1 < n, o, 1, 0, o, 1, 0, S + 96 * (k + 1 < n ? k + 1 : 0), 1, 0);
  u3072_coop_mul_mod(sm[grp], lane, act, o, 1, 0, o, 1, 0, num + num_pitch * k, 1, 0);
}
__global__ void __launch_bounds__(128) k_muhash_emit_hashes(const uint32_t* __restrict__ vals, size_t n, uint32_t* __restrict__ serialized, uint32_t* __restrict__ hashes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t r[96];
  u3072_canonical(r, vals + 96 * i, 1, 0);
  Blake2b h;
  b2b_init_muhash_finalize(h);
  for (int k = 0; k < 96; k++) { if (serialized) serialized[96 * i + k] = r[k]; b2b_u32(h, r[k]); }
  uint64_t d[4];
  b2b_final(h, d);
  for (int k = 0; k < 4; k++) { hashes[8 * i + 2 * k] = (uint32_t)d[k]; hashes[8 * i + 2 * k + 1] = (uint32_t)(d[k] >> 32); }
}
__global__ void k_u3072_canonicalize(uint32_t* __restrict__ vals, size_t pitch, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t r[96];
  u3072_canonical(r, vals + pitch * i, 1, 0);
  for (int k = 0; k < 96; k++) vals[pitch * i + k] = r[k];
}

// inclusive scan of n values (device array, pitch words apart) on stream st; tot: scratch for ceil(n/32) values
int kgv_mu_scan(kgv_ctx* ctx, uint32_t* vals, size_t pitch, size_t n, bool rev, uint32_t* tot, cudaStream_t st) {
  if (n <= 1) return KGV_OK;
  const size_t n_chunks = (n + KGV_SCAN_CHUNK - 1) / KGV_SCAN_CHUNK;
  k_u3072_scan_chunks<<<nblk(n_chunks, KGV_COOP_GROUPS), 128, 0, st>>>(vals, pitch, n, rev);
  CK(cudaGetLastError());
  ctx->launches++;
  if (n_chunks > 1) {
    k_u3072_scan_totals<<<1, 32, 0, st>>>(vals, pitch, n, rev, tot);
    CK(cudaGetLastError());
    k_u3072_scan_apply<<<nblk(n - KGV_SCAN_CHUNK, KGV_COOP_GROUPS), 128, 0, st>>>(vals, pitch, n, rev, tot);
    CK(cudaGetLastError());
    ctx->launches += 2;
  }
  return KGV_OK;
}

void kgv_mu_finalize_work::carve(kgv_carve& c, size_t n) {
  P = c.take<uint32_t>(n * 96); S = c.take<uint32_t>(n * 96); out = c.take<uint32_t>(n * 96);
  tot = c.take<uint32_t>((n + KGV_SCAN_CHUNK - 1) / KGV_SCAN_CHUNK * 96); inv = c.take<uint32_t>(3 * 96);
}
int kgv_mu_finalize_run(kgv_ctx* ctx, const uint32_t* dnum, const uint32_t* dden, size_t n, size_t pitch_words, const kgv_mu_finalize_work& w,
                        uint32_t* dser, uint32_t* dhashes, cudaStream_t st) {
  if (n == 0) return KGV_OK;
  uint32_t *P = w.P, *S = w.S, *out = w.out, *tot = w.tot, *inv = w.inv;
  CK(cudaMemcpy2DAsync(P, 384, dden, pitch_words * 4, 384, n, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(S, P, n * 384, cudaMemcpyDeviceToDevice, st));
  int rc = kgv_mu_scan(ctx, P, 96, n, false, tot, st);
  if (rc) return rc;
  rc = kgv_mu_scan(ctx, S, 96, n, true, tot, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(inv, P + 96 * (n - 1), 384, cudaMemcpyDeviceToDevice, st));
  k_u3072_inverse_one<<<1, 32, 0, st>>>(inv);
  CK(cudaGetLastError());
  k_muhash_divide_all<<<nblk(n, KGV_COOP_GROUPS), 128, 0, st>>>(dnum, pitch_words, P, S, inv + 96, n, out);
  CK(cudaGetLastError());
  k_muhash_emit_hashes<<<nblk(n, 128), 128, 0, st>>>(out, n, dser, dhashes);
  CK(cudaGetLastError());
  ctx->launches += 3;
  return KGV_OK;
}

extern "C" int kgv_muhash_finalize_batch(kgv_ctx* ctx, const uint8_t* numerators384, const uint8_t* denominators384, size_t n, size_t pitch_bytes, uint8_t* serialized384,
                                         uint8_t* hashes32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  // k_muhash_divide_all reads numerator k with 16-byte loads at numerators384 + k * pitch_bytes; the hash / serialize kernel stores words
  if (!numerators384 || !denominators384 || !hashes32 || pitch_bytes < 384 || (pitch_bytes & 15)) { ctx->err = "bad argument (pitch_bytes must be >= 384 and a multiple of 16)"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  bool dev;
  if (int rc = io.one_side("kgv_muhash_finalize_batch", {numerators384, denominators384, hashes32}, &dev)) return rc;
  // serialized384 is on its own side: its alignment is checked when it is device memory, whatever the side of the others
  if ((dev && (((uintptr_t)numerators384 & 15) || ((uintptr_t)hashes32 & 3))) || (serialized384 && io.is_device(serialized384) && ((uintptr_t)serialized384 & 3))) {
    ctx->err = "kgv_muhash_finalize_batch: device numerators384 must be 16-byte aligned, hashes32 and serialized384 4-byte aligned";
    return KGV_ERR_ARG;
  }
  // a strided host array is one contiguous span (the pitch interleaves numerators and denominators of MuHash records)
  const size_t span = (n - 1) * pitch_bytes + 384;
  kgv_mu_finalize_work w;
  int rc = kgv_reserve_carved(ctx, &ctx->d_mu, &ctx->d_mu_cap, [&](kgv_carve& c) { w.carve(c, n); });
  if (rc) return rc;
  const uint32_t *dnum, *dden;
  uint32_t *dh, *dser;
  io.in((const uint32_t*)numerators384, span, &dnum);
  io.in((const uint32_t*)denominators384, span, &dden);
  io.out((uint32_t*)hashes32, n * 32, &dh);
  io.out((uint32_t*)serialized384, n * 384, &dser);
  if ((rc = io.stage())) return rc;
  if ((rc = kgv_mu_finalize_run(ctx, dnum, dden, n, pitch_bytes / 4, w, dser, dh, ctx->stream))) return rc;
  return io.finish();
}

void kgv_mu_prefix_work::carve(kgv_carve& c, size_t n) { tot = c.take<uint32_t>((n + KGV_SCAN_CHUNK - 1) / KGV_SCAN_CHUNK * 96); }
int kgv_mu_prefix_combine_run(kgv_ctx* ctx, const uint32_t* dinit, uint32_t* v, size_t n, const kgv_mu_prefix_work& w, cudaStream_t st) {
  if (n == 0) return KGV_OK;
  if (dinit) {
    k_u3072_mul_first<<<1, 32, 0, st>>>(v, dinit, 2, 96);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  int rc = kgv_mu_scan(ctx, v, 192, n, false, w.tot, st);        // numerators
  if (rc) return rc;
  rc = kgv_mu_scan(ctx, v + 96, 192, n, false, w.tot, st);   // denominators
  if (rc) return rc;
  k_u3072_canonicalize<<<nblk(2 * n, 128), 128, 0, st>>>(v, 96, 2 * n);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

extern "C" int kgv_muhash_prefix_combine(kgv_ctx* ctx, const uint8_t* init768, uint8_t* values768, size_t n) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!values768) { ctx->err = "null argument"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (io.is_device(values768) && ((uintptr_t)values768 & 15)) { ctx->err = "kgv_muhash_prefix_combine: device values768 must be 16-byte aligned"; return KGV_ERR_ARG; }  // scanned in place with 16-byte loads
  kgv_mu_prefix_work w;
  uint32_t* dinit;
  int rc = kgv_reserve_carved(ctx, &ctx->d_mu, &ctx->d_mu_cap, [&](kgv_carve& c) { w.carve(c, n); dinit = c.take<uint32_t>(192); });
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  uint32_t* v;
  io.inout((uint32_t*)values768, n * 768, &v);
  if ((rc = io.stage())) return rc;
  if (init768) CK(cudaMemcpyAsync(dinit, init768, 768, io.is_device(init768) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  rc = kgv_mu_prefix_combine_run(ctx, init768 ? dinit : nullptr, v, n, w, st);
  if (rc) return rc;
  return io.finish();
}

// products of ranges of level-0 elements (kgv_replay_muhash): E has `stride` elements; flags[flag_index[j]] != 0 selects element j
int kgv_mu_range_products(kgv_ctx* ctx, const uint32_t* E, size_t stride, const uint8_t* flags, const uint32_t* flag_index, const uint32_t* lo, const uint32_t* hi, uint32_t n_segs,
                          uint32_t* out, size_t out_pitch_words, cudaStream_t st) {
  if (n_segs == 0) return KGV_OK;
  k_u3072_range_product<<<nblk(n_segs, KGV_COOP_GROUPS), 128, 0, st>>>(E, stride, flags, flag_index, lo, hi, n_segs, out, out_pitch_words);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

int kgv_mu_canonicalize(kgv_ctx* ctx, uint32_t* vals, size_t pitch_words, size_t n, cudaStream_t st) {
  if (!n) return KGV_OK;
  k_u3072_canonicalize<<<nblk(n, 128), 128, 0, st>>>(vals, pitch_words, n);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}
