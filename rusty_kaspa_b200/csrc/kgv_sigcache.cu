// kgv_sigcache.cu — the SigCache analogue: a device-resident, bounded table of signature verdicts.
//
// Reference: Cache<SigCacheKey, bool> (crypto/txscript/src/caches.rs:14-55; key = (signature, public key, message),
// crypto/txscript/src/lib.rs:72-76), consulted by check_schnorr_signature / check_ecdsa_signature AFTER the key and signature parsed
// (lib.rs:582-603, 618-638: parse errors never reach the cache), filled with true AND false verdicts, bounded at 10 000 entries
// (consensus/src/processes/transaction_validator/mod.rs:48) with random eviction when full (caches.rs:49-51), shared by all clones of the
// TransactionValidator (mempool validation, template building and block validation see each other's verdicts), counters :57-93.
// It changes speed, never results - the same holds here:
//   key      BLAKE2b-256(kind || sig64 || pk || msg32): collision-free for any purpose an attacker could have, so a hit returns the
//            verdict of exactly that triple
//   table    power-of-two slots of (32-byte digest, 1 verdict byte); an entry lives in one of the PROBE slots after its home slot
//   lookup   one thread per candidate pair, before the verify kernels; hits are answered from the table, the MISSES are compacted into an
//            index list on the device and only those go through the (index-driven) verify kernels
//   insert   after verification, verdicts 0 / 1 of the misses; when all PROBE slots are taken one of them, picked by a hash of the
//            digest, is overwritten (random eviction, bounded memory)
// Writers mark a slot busy, write the digest, fence, then publish the verdict; readers re-read the verdict byte after comparing the
// digest, so concurrent use by several contexts (streams) never yields a verdict that belongs to another triple.
#include "kgv_internal.h"
#include "kgv_blake2b.cuh"

#include <cstdio>

using namespace kgv;

#define SC_PROBE 8
#define SC_EMPTY 0u
#define SC_BUSY 0xFFu  // verdicts are stored as 1 (invalid) / 2 (valid)

struct kgv_sigcache {
  kgv_ctx* owner = nullptr;
  uint64_t* digests = nullptr;  // capacity x 4 words
  uint8_t* val = nullptr;       // capacity bytes (accessed through 32-bit CAS on the containing word)
  uint64_t mask = 0;
  unsigned long long* counters = nullptr;  // [0] hits (get_counts), [1] inserts (insert_counts), [2] lookups, [3] evictions
};

__device__ __forceinline__ uint32_t val_load(const uint8_t* val, uint64_t i) { return *(volatile const uint8_t*)(val + i); }
// CAS on one byte of the verdict array through its aligned 32-bit word
__device__ __forceinline__ bool val_cas(uint8_t* val, uint64_t i, uint32_t expect, uint32_t desired) {
  uint32_t* w = (uint32_t*)(val + (i & ~(uint64_t)3));
  const uint32_t sh = (uint32_t)(i & 3) * 8;
  uint32_t old = *(volatile uint32_t*)w;
  for (;;) {
    if (((old >> sh) & 0xFFu) != expect) return false;
    const uint32_t nw = (old & ~(0xFFu << sh)) | (desired << sh);
    const uint32_t got = atomicCAS(w, old, nw);
    if (got == old) return true;
    old = got;
  }
}

__global__ void __launch_bounds__(128) k_sc_lookup(const uint64_t* __restrict__ tab, const uint8_t* __restrict__ val, uint64_t mask, const uint8_t* __restrict__ pk,
                                                   const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig, size_t n, uint32_t pk_len, uint8_t* __restrict__ status,
                                                   uint64_t* __restrict__ digests, unsigned long long* __restrict__ counters) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = false;
  if (i < n) {
    Blake2b h;
    b2b_init(h, B2B_UNKEYED);
    b2b_u8(h, pk_len);  // 32: Schnorr, 33: ECDSA
    b2b_bytes(h, sig + 64 * i, 64);
    b2b_bytes(h, pk + (size_t)pk_len * i, pk_len);
    b2b_bytes(h, msg + 32 * i, 32);
    uint64_t d[4];
    b2b_final(h, d);
#pragma unroll
    for (int k = 0; k < 4; k++) digests[4 * i + k] = d[k];
    uint32_t verdict = 0xFF;
    const uint64_t home = d[0] & mask;
    for (int p = 0; p < SC_PROBE && !hit; p++) {
      const uint64_t s = (home + p) & mask;
      const uint32_t v = val_load(val, s);
      if (v == SC_EMPTY || v == SC_BUSY) continue;
      const uint64_t* e = tab + 4 * s;
      const bool eq = __ldcg(e) == d[0] && __ldcg(e + 1) == d[1] && __ldcg(e + 2) == d[2] && __ldcg(e + 3) == d[3];
      if (eq && val_load(val, s) == v) { hit = true; verdict = v - 1; }
    }
    status[i] = (uint8_t)verdict;
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
  const unsigned a = __ballot_sync(0xFFFFFFFFu, i < n);
  if ((threadIdx.x & 31) == 0) {
    if (m) atomicAdd(&counters[0], (unsigned long long)__popc(m));
    if (a) atomicAdd(&counters[2], (unsigned long long)__popc(a));
  }
}
// ordered compaction of the misses (status == 0xFF) into an index list: one block, chunked like the item-offset scan
__global__ void __launch_bounds__(1024) k_sc_compact(const uint8_t* __restrict__ status, size_t n, uint32_t* __restrict__ index, uint32_t* __restrict__ n_miss) {
  __shared__ uint32_t part[1024];
  const size_t per = (n + 1023) / 1024;
  const size_t a = (size_t)threadIdx.x * per, b = a + per < n ? a + per : n;
  uint32_t s = 0;
  for (size_t i = a; i < b; i++) s += status[i] == 0xFF;
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    uint32_t t = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  uint32_t run = part[threadIdx.x] - s;
  for (size_t i = a; i < b; i++) if (status[i] == 0xFF) index[run++] = (uint32_t)i;
  if (threadIdx.x == 1023) *n_miss = part[1023];
}
__global__ void __launch_bounds__(128) k_sc_insert(uint64_t* __restrict__ tab, uint8_t* __restrict__ val, uint64_t mask, const uint8_t* __restrict__ status,
                                                   const uint64_t* __restrict__ digests, const uint32_t* __restrict__ index, const uint32_t* __restrict__ n_miss,
                                                   unsigned long long* __restrict__ counters) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *n_miss) return;
  const uint32_t i = index[j];
  const uint32_t st = status[i];
  if (st > 1) return;  // parse errors are recomputed, as in the reference (lib.rs:582-583, 618-619 run before the cache)
  uint64_t d[4];
#pragma unroll
  for (int k = 0; k < 4; k++) d[k] = digests[4 * (size_t)i + k];
  const uint64_t home = d[0] & mask;
  uint64_t slot = ~0ull;
  for (int p = 0; p < SC_PROBE; p++) {
    const uint64_t s = (home + p) & mask;
    if (val_load(val, s) == SC_EMPTY && val_cas(val, s, SC_EMPTY, SC_BUSY)) { slot = s; break; }
  }
  if (slot == ~0ull) {  // full neighbourhood: evict one of its entries, chosen by bits of the digest the home slot does not depend on
    const uint64_t s = (home + ((d[1] >> 17) % SC_PROBE)) & mask;
    const uint32_t v = val_load(val, s);
    if (v == SC_BUSY || !val_cas(val, s, v, SC_BUSY)) return;  // somebody else is writing there: give up, a cache may forget
    slot = s;
    atomicAdd(&counters[3], 1ull);
  }
  uint64_t* e = tab + 4 * slot;
#pragma unroll
  for (int k = 0; k < 4; k++) __stcg(e + k, d[k]);
  __threadfence();
  val_cas(val, slot, SC_BUSY, st + 1);
  atomicAdd(&counters[1], 1ull);
}

extern "C" int kgv_sigcache_create(kgv_ctx* ctx, uint64_t capacity, kgv_sigcache** out) {
  if (!ctx || !out) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  uint64_t cap = 64;
  while (cap < capacity) cap <<= 1;
  kgv_sigcache* c = new kgv_sigcache();
  c->owner = ctx;
  c->mask = cap - 1;
  cudaError_t e = cudaMalloc((void**)&c->digests, cap * 32);
  if (e == cudaSuccess) e = cudaMalloc((void**)&c->val, cap);
  if (e == cudaSuccess) e = cudaMalloc((void**)&c->counters, 8 * sizeof(unsigned long long));
  if (e != cudaSuccess) {
    ctx->err = std::string("cudaMalloc failed for the signature cache: ") + cudaGetErrorString(e);
    (void)cudaGetLastError();
    if (c->digests) cudaFree(c->digests);
    if (c->val) cudaFree(c->val);
    delete c;
    return KGV_ERR_NOMEM;
  }
  CK(cudaMemsetAsync(c->val, 0, cap, ctx->stream));
  CK(cudaMemsetAsync(c->counters, 0, 8 * sizeof(unsigned long long), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *out = c;
  return KGV_OK;
}
extern "C" void kgv_sigcache_destroy(kgv_sigcache* c) {
  if (!c) return;
  if (c->owner) { cudaSetDevice(c->owner->device); cudaStreamSynchronize(c->owner->stream); if (c->owner->sigcache == c) c->owner->sigcache = nullptr; }
  cudaFree(c->digests); cudaFree(c->val); cudaFree(c->counters);
  delete c;
}
extern "C" int kgv_sigcache_clear(kgv_ctx* ctx, kgv_sigcache* c) {
  if (!ctx || !c) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemsetAsync(c->val, 0, c->mask + 1, ctx->stream));
  return KGV_OK;
}
extern "C" int kgv_sigcache_counters(kgv_ctx* ctx, kgv_sigcache* c, uint64_t* hits, uint64_t* inserts, uint64_t* lookups, uint64_t* evictions) {
  if (!ctx || !c) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  for (const auto& [what, p] : {std::pair<const char*, const void*>{"hits", hits}, {"inserts", inserts}, {"lookups", lookups}, {"evictions", evictions}})
    if (int rc = kgv_host_only(ctx, "kgv_sigcache_counters", what, p)) return rc;
  CK(cudaSetDevice(ctx->device));
  unsigned long long h[4];
  CK(cudaMemcpyAsync(h, c->counters, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (hits) *hits = h[0];
  if (inserts) *inserts = h[1];
  if (lookups) *lookups = h[2];
  if (evictions) *evictions = h[3];
  return KGV_OK;
}
extern "C" int kgv_set_sigcache(kgv_ctx* ctx, kgv_sigcache* c) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (c && c->owner->device != ctx->device) { ctx->err = "the signature cache lives on another device"; return KGV_ERR_ARG; }
  ctx->sigcache = c;
  return KGV_OK;
}

int kgv_sigcache_lookup(kgv_ctx* ctx, kgv_sigcache* c, const uint8_t* pk, const uint8_t* msg, const uint8_t* sig, size_t n, bool ecdsa, uint8_t* status, uint8_t* digests,
                        uint32_t* miss_index, uint32_t* n_miss_dev, cudaStream_t st) {
  if (!n) return KGV_OK;
  k_sc_lookup<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(c->digests, c->val, c->mask, pk, msg, sig, n, ecdsa ? 33u : 32u, status, (uint64_t*)digests, c->counters);
  CK(cudaGetLastError());
  k_sc_compact<<<1, 1024, 0, st>>>(status, n, miss_index, n_miss_dev);
  CK(cudaGetLastError());
  ctx->launches += 2;
  return KGV_OK;
}
int kgv_sigcache_insert(kgv_ctx* ctx, kgv_sigcache* c, const uint8_t* status, const uint8_t* digests, const uint32_t* miss_index, const uint32_t* n_miss_dev, size_t n_max,
                        cudaStream_t st) {
  if (!n_max) return KGV_OK;
  k_sc_insert<<<(unsigned)((n_max + 127) / 128), 128, 0, st>>>(c->digests, c->val, c->mask, status, (const uint64_t*)digests, miss_index, n_miss_dev, c->counters);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}
