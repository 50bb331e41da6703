// kgv_headers.cu — kgv_hash_headers and kgv_validate_headers_in_isolation: the block hash, proof of work and block level of a batch of
// headers (HeaderProcessor::validate_header_in_isolation, consensus/src/pipeline/header_processor/pre_ghostdag_validation.rs:17-24), and
// the kgv_debug_pow_matrix hook.  The per-header pieces are in kgv_pow.cuh.
//   k_header_hash      one thread per header: the block hash and / or the pre-PoW hash
//   k_header_validate  one 64-thread CTA per header:
//                        warp 0 lane 0   pre-PoW hash, then the xoshiro256++ draws (sequential by nature: 256 per matrix)
//                        warp 1 lane 0   block hash, then the cSHAKE256 "ProofOfWorkHash" of the pre-PoW hash
//                        all 64 threads  compute_rank with one matrix column per thread (the f64 matrix, 33 KB, in shared memory),
//                                        repeated while the rank is below 64; then one heavy-hash row sum per thread
//                        thread 0        kHeavyHash, target, level, the isolation rules and the result record
#include "kgv_internal.h"
#include "kgv_pow.cuh"

#include <cstdio>

using namespace kgv;

static_assert(sizeof(kgv_header) == 208, "kgv_header is 208 bytes");
static_assert(sizeof(kgv_header_rules) == 32, "kgv_header_rules is 32 bytes");
static_assert(sizeof(kgv_header_result) == 24, "kgv_header_result is 24 bytes");


constexpr int HDR_HASH_THREADS = 128;
constexpr int HDR_CTA = 64;

struct HeaderArena {
  const kgv_header* h;
  const uint8_t* parents;
  const uint32_t* level_len;
  uint64_t n, n_parents, n_level_entries;
  unsigned int* bad;  // set when a header's arena range leaves the arena
};

__global__ void __launch_bounds__(HDR_HASH_THREADS) k_header_hash(HeaderArena ar, uint64_t* hash, uint64_t* pre) {
  const uint64_t k = (uint64_t)blockIdx.x * HDR_HASH_THREADS + threadIdx.x;
  if (k >= ar.n) return;
  const kgv_header h = ar.h[k];
  uint64_t np;
  if (!header_ranges_ok(h, ar.level_len, ar.n_level_entries, ar.n_parents, &np)) { atomicOr(ar.bad, 1u); return; }
  const uint8_t* par = ar.parents + 32 * h.parents_off;
  const uint32_t* lens = ar.level_len + h.levels_off;
  uint64_t d[4];
  if (hash) {
    header_hash(h, par, lens, h.nonce, h.timestamp, d);
#pragma unroll
    for (int w = 0; w < 4; w++) hash[4 * k + w] = d[w];
  }
  if (pre) {
    header_hash(h, par, lens, 0, 0, d);
#pragma unroll
    for (int w = 0; w < 4; w++) pre[4 * k + w] = d[w];
  }
}

struct PowSmem {
  double a[64 * RANK_STRIDE];
  uint64_t w[256];     // the drawn matrix, matrix_draw layout
  uint64_t pre[4], pw[4];
  uint32_t rows[64];
  uint32_t ballot[2];
  uint32_t ok;
};

// the matrix in s.w, as f64 into s.a (all threads)
__device__ __forceinline__ void load_nibble_matrix(PowSmem& s) {
  for (int e = threadIdx.x; e < 64 * 64; e += HDR_CTA) s.a[(e >> 6) * RANK_STRIDE + (e & 63)] = (double)matrix_elem(s.w, e >> 6, e & 63);
}

// compute_rank of s.a, one column per thread; every thread returns the rank
__device__ uint32_t cta_rank(PowSmem& s) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  uint64_t sel = 0;
  uint32_t rank = 0;
  for (int i = 0; i < 64; i++) {
    // the first unselected row with |a[j][i]| > eps: row t asks, the lowest asking row wins
    const bool cand = !((sel >> t) & 1) && fabs(s.a[t * RANK_STRIDE + i]) > RANK_EPS;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, cand);
    if (lane == 0) s.ballot[warp] = b;
    __syncthreads();
    const uint64_t both = (uint64_t)s.ballot[0] | (uint64_t)s.ballot[1] << 32;
    __syncthreads();  // ballot is rewritten by the next step
    if (!both) continue;
    const int j = __ffsll((long long)both) - 1;
    rank++;
    sel |= 1ull << j;
    if (t > i) rank_column(s.a, i, j, t);
    __syncthreads();
  }
  return rank;
}

// Matrix::generate from s.pre (seed words): leaves the matrix in s.w; returns the number of matrices drawn
__device__ uint32_t cta_generate(PowSmem& s) {
  Xoshiro x;
  if (threadIdx.x == 0) xoshiro_seed(x, s.pre);
  uint32_t tries = 0;
  for (;;) {
    if (threadIdx.x == 0) matrix_draw(x, s.w);
    __syncthreads();
    load_nibble_matrix(s);
    __syncthreads();
    tries++;
    if (cta_rank(s) == 64) return tries;
  }
}

struct ValidateArgs {
  HeaderArena ar;
  kgv_header_rules r;
  kgv_header_result* res;
  uint64_t* hash;  // may be null
  uint64_t* pow;   // may be null
};

__global__ void __launch_bounds__(HDR_CTA) k_header_validate(ValidateArgs a) {
  __shared__ PowSmem s;
  const uint64_t k = blockIdx.x;
  const kgv_header h = a.ar.h[k];
  const int t = threadIdx.x;
  if (t == 0) {
    uint64_t np;
    s.ok = header_ranges_ok(h, a.ar.level_len, a.ar.n_level_entries, a.ar.n_parents, &np);
    if (!s.ok) atomicOr(a.ar.bad, 1u);
  }
  __syncthreads();
  if (!s.ok) return;
  const uint8_t* par = a.ar.parents + 32 * h.parents_off;
  const uint32_t* lens = a.ar.level_len + h.levels_off;
  if (t == 0) header_hash(h, par, lens, 0, 0, s.pre);
  if (t == 32 && a.hash) {
    uint64_t d[4];
    header_hash(h, par, lens, h.nonce, h.timestamp, d);
#pragma unroll
    for (int w = 0; w < 4; w++) a.hash[4 * k + w] = d[w];
  }
  __syncthreads();
  if (t == 32) pow_hash(s.pre, h.timestamp, h.nonce, s.pw);  // beside the first draws of thread 0
  cta_generate(s);
  s.rows[t] = heavy_row_sum(s.w, t, s.pw);
  __syncthreads();
  if (t != 0) return;
  uint64_t pw[4], target[4];
  heavy_finish(s.rows, s.pw, pw);
  compact_target(h.bits, target);
  const bool genesis = h.n_levels == 0;
  const bool passed = genesis || u256_le(pw, target);
  const uint32_t level = genesis ? a.r.max_block_level : level_from_pow(pw, a.r.max_block_level);
  kgv_header_result out;
  header_rules(h, par, genesis ? 0u : lens[0], a.r, passed, out);
  out.level = (uint8_t)level;
  out.pow_passed = passed;
  out.pad_ = 0;
  a.res[k] = out;
  if (a.pow) {
#pragma unroll
    for (int w = 0; w < 4; w++) a.pow[4 * k + w] = pw[w];
  }
}

// kgv_debug_pow_matrix: op 0 ranks caller matrices (u16), op 1 generates from seeds
__global__ void __launch_bounds__(HDR_CTA) k_pow_matrix_debug(int op, const uint8_t* in, uint8_t* out) {
  __shared__ PowSmem s;
  const uint64_t k = blockIdx.x;
  const int t = threadIdx.x;
  if (op == 0) {
    const uint16_t* m = (const uint16_t*)(in + k * 8192);
    for (int e = t; e < 4096; e += HDR_CTA) s.a[(e >> 6) * RANK_STRIDE + (e & 63)] = (double)m[e];
    __syncthreads();
    const uint32_t r = cta_rank(s);
    if (t == 0) ((uint32_t*)out)[k] = r;
    return;
  }
  if (t < 4) s.pre[t] = ((const uint64_t*)(in + 32 * k))[t];
  __syncthreads();
  const uint32_t tries = cta_generate(s);
  uint8_t* o = out + k * 4100;
  for (int e = t; e < 4096; e += HDR_CTA) o[e] = (uint8_t)matrix_elem(s.w, e >> 6, e & 63);
  if (t == 0) memcpy(o + 4096, &tries, 4);
}

// ---- C ABI ------------------------------------------------------------------------------------------------------------------------

// Declares the header arrays and the arena-range flag of a call; its HeaderArena is complete after io.stage() (ar->bad: clear it)
static void declare_headers(kgv_io& io, const kgv_header* headers, size_t n, const uint8_t* parents32, size_t n_parents, const uint32_t* level_len,
                            size_t n_level_entries, unsigned int* bad, HeaderArena* ar) {
  ar->n = n; ar->n_parents = n_parents; ar->n_level_entries = n_level_entries;
  io.in(headers, n * sizeof(kgv_header), &ar->h);
  io.in(n_parents ? parents32 : nullptr, n_parents * 32, &ar->parents);
  io.in(n_level_entries ? level_len : nullptr, n_level_entries * 4, &ar->level_len);
  io.out(bad, 4, &ar->bad);  // a host scalar: finish() always waits for the call
}

// the refusals shared by the two calls: null or mixed arrays, device arrays not 8-byte aligned
static int check_headers(kgv_ctx* ctx, kgv_io& io, const char* call, const kgv_header* headers, const uint8_t* parents32, size_t n_parents,
                         const uint32_t* level_len, size_t n_level_entries, const void* o0, const void* o1, const void* o2) {
  if ((n_parents && !parents32) || (n_level_entries && !level_len)) return fail_arg(ctx, "null argument");
  bool dev;
  if (int rc = io.one_side(call, {headers, n_parents ? parents32 : nullptr, n_level_entries ? level_len : nullptr, o0, o1, o2}, &dev)) return rc;
  const uintptr_t a = (uintptr_t)headers | (uintptr_t)parents32 | (uintptr_t)o0 | (uintptr_t)o1 | (uintptr_t)o2;
  if (dev && ((a & 7) || (n_level_entries && ((uintptr_t)level_len & 3)))) return fail_arg(ctx, (std::string(call) + ": device headers, parents32 and outputs must be 8-byte aligned, level_len 4-byte aligned").c_str());
  return KGV_OK;
}

// waits for the call and reports an arena range outside the arena
static int finish_headers(kgv_ctx* ctx, kgv_io& io, const char* call, const unsigned int& bad) {
  if (int rc = io.finish()) return rc;
  return bad ? fail_arg(ctx, (std::string(call) + ": a header's levels_off / parents_off range leaves the arena").c_str()) : KGV_OK;
}

// hashing::header::hash and hash_override_nonce_time(h, 0, 0) (consensus/core/src/hashing/header.rs:7-35)
extern "C" int kgv_hash_headers(kgv_ctx* ctx, const kgv_header* headers, size_t n, const uint8_t* parents32, size_t n_parents, const uint32_t* level_len,
                                size_t n_level_entries, uint8_t* hash32, uint8_t* pre_pow32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!headers || (!hash32 && !pre_pow32)) return fail_arg(ctx, "null argument");
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  int rc = check_headers(ctx, io, "kgv_hash_headers", headers, parents32, n_parents, level_len, n_level_entries, hash32, pre_pow32, nullptr);
  if (rc) return rc;
  HeaderArena ar;
  unsigned int bad = 0;
  uint64_t *dh, *dp;
  declare_headers(io, headers, n, parents32, n_parents, level_len, n_level_entries, &bad, &ar);
  io.out((uint64_t*)hash32, 32 * n, &dh);
  io.out((uint64_t*)pre_pow32, 32 * n, &dp);
  if ((rc = io.stage())) return rc;
  CK(cudaMemsetAsync(ar.bad, 0, 4, ctx->stream));
  k_header_hash<<<(unsigned)((n + HDR_HASH_THREADS - 1) / HDR_HASH_THREADS), HDR_HASH_THREADS, 0, ctx->stream>>>(ar, dh, dp);
  CK(cudaGetLastError());
  ctx->launches++;
  return finish_headers(ctx, io, "kgv_hash_headers", bad);
}

// validate_header_in_isolation (pre_ghostdag_validation.rs:17-24) with check_pow_and_calc_block_level (:102-106) for every header
extern "C" int kgv_validate_headers_in_isolation(kgv_ctx* ctx, const kgv_header* headers, size_t n, const uint8_t* parents32, size_t n_parents,
                                                 const uint32_t* level_len, size_t n_level_entries, const kgv_header_rules* rules,
                                                 kgv_header_result* results, uint8_t* hash32, uint8_t* pow32) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!headers || !rules || !results) return fail_arg(ctx, "null argument");
  if (int rc = kgv_host_only(ctx, "kgv_validate_headers_in_isolation", "rules", rules)) return rc;
  if (rules->max_block_level > 255) return fail_arg(ctx, "max_block_level is a BlockLevel (u8)");
  if (n > 0x7FFFFFFFull) return fail_arg(ctx, "at most 2^31 - 1 headers per call");
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  int rc = check_headers(ctx, io, "kgv_validate_headers_in_isolation", headers, parents32, n_parents, level_len, n_level_entries, results, hash32, pow32);
  if (rc) return rc;
  ValidateArgs a;
  unsigned int bad = 0;
  declare_headers(io, headers, n, parents32, n_parents, level_len, n_level_entries, &bad, &a.ar);
  io.out(results, n * sizeof(kgv_header_result), &a.res);
  io.out((uint64_t*)hash32, 32 * n, &a.hash);
  io.out((uint64_t*)pow32, 32 * n, &a.pow);
  if ((rc = io.stage())) return rc;
  CK(cudaMemsetAsync(a.ar.bad, 0, 4, ctx->stream));
  a.r = *rules;
  k_header_validate<<<(unsigned)n, HDR_CTA, 0, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches++;
  return finish_headers(ctx, io, "kgv_validate_headers_in_isolation", bad);
}

extern "C" int kgv_debug_pow_matrix(kgv_ctx* ctx, int op, const uint8_t* in, size_t n, uint8_t* out) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!in || !out || (op != 0 && op != 1)) return fail_arg(ctx, "null argument or unknown op");
  if (n > (1u << 20)) return fail_arg(ctx, "at most 2^20 matrices per call");
  if (kgv_ptr_is_device(in) || kgv_ptr_is_device(out)) return fail_arg(ctx, "host pointers only");
  CK(cudaSetDevice(ctx->device));
  const size_t in_b = n * (op == 0 ? 8192 : 32), out_b = n * (op == 0 ? 4 : 4100);
  int rc = kgv_reserve(ctx, &ctx->d_in, &ctx->d_in_cap, in_b);
  if (rc) return rc;
  rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, out_b);
  if (rc) return rc;
  CK(cudaMemcpyAsync(ctx->d_in, in, in_b, cudaMemcpyHostToDevice, ctx->stream));
  k_pow_matrix_debug<<<(unsigned)n, HDR_CTA, 0, ctx->stream>>>(op, ctx->d_in, ctx->d_out);
  CK(cudaGetLastError());
  ctx->launches++;
  CK(cudaMemcpyAsync(out, ctx->d_out, out_b, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}
