// kgv_lib.cu — kernels and C ABI of libkgv.so (see include/kgv.h).
//
// Hand-written CUDA for sm_90a (H100).  No CPU fallback: every entry point needs a CUDA device.
#include "../../include/kgv.h"
#include "kgv_internal.h"
#include "kgv_verify.cuh"
#include "kgv_lanes.cuh"

#include <cuda_runtime.h>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>

using namespace kgv;

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
// per-thread table in shared memory, word-major / thread-minor: every access of a warp hits 32
// consecutive banks whatever entry each lane selects
struct SmemTab {
  uint32_t* base;  // smem + threadIdx.x
  __device__ __forceinline__ void put(int e, int w, uint32_t v) { base[(e * 16 + w) * KGV_BLOCK] = v; }
  __device__ __forceinline__ uint32_t get(int e, int w) const { return base[(e * 16 + w) * KGV_BLOCK]; }
  // the comb ladder's staging (ecmult_joint) uses the same 512 bytes as 32 chunks of 16 bytes, chunk-major / thread-minor: a warp's
  // 16-byte copies and reads of one chunk cover 512 consecutive bytes, free of bank conflicts.  Chunk c of slot s: 4s + c.
  __device__ __forceinline__ uint4* chunk(int q) const { return reinterpret_cast<uint4*>(base - threadIdx.x) + q * KGV_BLOCK + threadIdx.x; }
};
__device__ __forceinline__ void stage_fetch(SmemTab& tab, int s, const uint32_t* entry) {
#pragma unroll
  for (int c = 0; c < 4; c++) {
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(tab.chunk(4 * s + c));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(entry + 4 * c) : "memory");
  }
}
__device__ __forceinline__ void stage_commit(SmemTab&) { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void stage_wait(SmemTab&) { asm volatile("cp.async.wait_group 7;" ::: "memory"); }
__device__ __forceinline__ void stage_get(SmemTab& tab, int s, fe& x, fe& y) {
  const uint4 a = *tab.chunk(4 * s), b = *tab.chunk(4 * s + 1), c = *tab.chunk(4 * s + 2), d = *tab.chunk(4 * s + 3);
  x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
  y.v[0] = c.x; y.v[1] = c.y; y.v[2] = c.z; y.v[3] = c.w; y.v[4] = d.x; y.v[5] = d.y; y.v[6] = d.z; y.v[7] = d.w;
}

// 256-bit read-only load: sm_90 has no 256-bit LDG, so two 128-bit loads of the same 32-byte sector, issued back to back
__device__ __forceinline__ void ldg256(uint32_t* w, const void* p) {
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
               : "l"(p));
}
// streaming variant for the signature triples (read once)
__device__ __forceinline__ void ldg256_stream(uint32_t* w, const void* p) {
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
               : "l"(p));
}

// generator table entry: 64 bytes, 64-byte aligned: two 256-bit loads
struct GLoadDev {
  __device__ __forceinline__ void operator()(fe& x, fe& y, const uint32_t* entry) const {
    ldg256(x.v, entry);
    ldg256(y.v, entry + 8);
  }
};

// 32 big-endian bytes -> 8 numeric words (w[0] most significant)
template <bool ALIGNED>
__device__ __forceinline__ void load_be32(uint32_t* w, const uint8_t* p) {
  if (ALIGNED) {
    ldg256_stream(w, p);
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = bswap32(w[i]);
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++)
      w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | (uint32_t)p[4 * i + 3];
  }
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_build_gtab(uint32_t* __restrict__ gtab) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 8u * 65536u) return;
  uint32_t v = t & 0xFFFFu;
  uint32_t which = t >> 16;
  uint32_t* out = gtab + (size_t)t * 16;
  if (v == 0) {
#pragma unroll
    for (int i = 0; i < 16; i++) out[i] = 0;
    return;
  }
  fe bx, by, x, y;
  gtab_base(bx, by, (int)which);
  gtab_entry(x, y, v, bx, by);
#pragma unroll
  for (int i = 0; i < 8; i++) { out[i] = x.v[i]; out[8 + i] = y.v[i]; }
}

// ---- per-launch key cache: the key part of a verification done once per distinct public key of a verify launch ----
// Records per launch at most (2^17 x 8320 B = 1.09 GB of comb-form records, 2^17 x 560 B = 73 MB of plain ones).
#define KGV_KEY_RECORDS_MAX (1u << 17)
// Fewest uses per key on average for comb records: the comb's preparation (~1 800 products per key against ~400, ~2 700 with the joint
// table, ~2 200 for the comb-form record that keeps only P and the joint table: 2.24 ms for 70 794 keys against 2.99 ms) must be paid
// back by its shorter ladder (~700, with the joint table ~1 000 products fewer per verify); measured +20 % at 10 uses per key before the
// joint table and faster still with it at 8 to 50 uses (DESIGN.md §5), not below.  Not re-tuned for the cheaper preparation.
#ifndef KGV_COMB_USES
#define KGV_COMB_USES 8
#endif
enum { KGV_KEYS_INLINE = 0, KGV_KEYS_PLAIN = 1, KGV_KEYS_COMB = 2 };
// The form of a launch's key part, uniform over the launch: records when its keys are used twice on average (at most n/2 distinct keys)
// and fit the cap; then EVERY key has one.  A warp pays for the inline key path of any of its lanes, so records for the repeated keys
// alone leave singleton lanes costing whole warps; a batch of mostly distinct keys makes no records at all and pays only the dedup pass.
// Comb-form records (key_joint_record_build, ecmult_joint) when the keys are used at least KGV_COMB_USES times on average, plain ones (key_rec_build) below.
// Host-callable too: kgv_debug_key_form reports the form a launch took by this same rule.
__host__ __device__ __forceinline__ int key_form(uint32_t n_rec, size_t n) {
  if (n_rec > KGV_KEY_RECORDS_MAX || 2 * (size_t)n_rec > n) return KGV_KEYS_INLINE;
  return (size_t)KGV_COMB_USES * n_rec <= n ? KGV_KEYS_COMB : KGV_KEYS_PLAIN;
}

// Slot of the open-addressed key table: key = fingerprint << 32 | (representative item + 1), 0 = empty; rec = the key's record + 1.
struct KeySlot {
  unsigned long long key;
  uint32_t rec, unused_;
};
struct KeyCacheView {
  const KeySlot* table;
  const uint32_t* item_slot;  // item -> table slot (only the items the launch verifies are set)
  const uint32_t* recs;       // records, KGV_KR_WORDS or KGV_JR_WORDS words each
  const uint32_t* n_rec;      // distinct keys of the launch; nullptr: no key cache
  // the key source of item i: its record and the launch's form, or no record (the launch makes none)
  __device__ __forceinline__ KeySrc key_of(size_t i, size_t n) const {
    const int f = n_rec ? key_form(*n_rec, n) : KGV_KEYS_INLINE;
    if (f == KGV_KEYS_INLINE) return KeySrc{nullptr, false};
    const bool comb = f == KGV_KEYS_COMB;
    return KeySrc{recs + (size_t)(table[item_slot[i]].rec - 1) * (comb ? KGV_JR_WORDS : KGV_KR_WORDS), comb};
  }
};

// the key of item i: 8 big-endian words of x (+ the tag byte as word 8 for ECDSA; 33-byte stride, never word aligned)
template <bool ALIGNED, bool ECDSA>
__device__ __forceinline__ void key_words(uint32_t* w, const uint8_t* pk, size_t i) {
  if (ECDSA) {
    const uint8_t* kp = pk + 33 * i;
    w[8] = kp[0];
    load_be32<false>(w, kp + 1);
  } else {
    load_be32<ALIGNED>(w, pk + 32 * i);
  }
}
__device__ __forceinline__ uint64_t key_hash(const uint32_t* w, int nw) {
  uint64_t h = 0x9E3779B97F4A7C15ull;
  for (int k = 0; k < nw; k++) {
    h = (h ^ w[k]) * 0xFF51AFD7ED558CCDull;
    h ^= h >> 32;
  }
  h ^= h >> 33; h *= 0xC4CEB9FE1A85EC53ull; h ^= h >> 33;
  return h;
}

// One thread per item: find or claim the key's slot; a claimed slot gets the next record index.  Whichever item's atomicCAS claims the
// slot becomes its representative: the record depends on the key bytes alone.  Once the launch has more keys than records allow (key_form),
// the remaining items stop (the verify kernels then take the inline key path for every item).
template <bool ALIGNED, bool ECDSA>
__global__ void __launch_bounds__(256) k_key_dedup(const uint8_t* __restrict__ pk, size_t n_arg, const uint32_t* __restrict__ index,
                                                   const uint32_t* __restrict__ n_dev, KeySlot* __restrict__ table, uint32_t mask,
                                                   uint32_t* __restrict__ item_slot, uint32_t* __restrict__ rec_rep, uint32_t* n_rec) {
  const size_t n = n_dev ? (size_t)*n_dev : n_arg;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n || key_form(*(volatile uint32_t*)n_rec, n) == KGV_KEYS_INLINE) return;
  const size_t i = index ? index[t] : t;
  const int nw = ECDSA ? 9 : 8;
  uint32_t w[9];
  key_words<ALIGNED, ECDSA>(w, pk, i);
  const uint64_t h = key_hash(w, nw);
  const unsigned long long mine = (h & 0xFFFFFFFF00000000ull) | (uint64_t)(i + 1);
  uint32_t s = (uint32_t)h & mask;
  bool won = false;
  for (;;) {
    unsigned long long cur = atomicCAS(&table[s].key, 0ull, mine);
    if (cur == 0) { won = true; break; }
    if ((cur >> 32) == (mine >> 32)) {
      uint32_t v[9];
      key_words<ALIGNED, ECDSA>(v, pk, (uint32_t)cur - 1);
      bool eq = true;
      for (int k = 0; k < nw; k++) eq = eq && v[k] == w[k];
      if (eq) break;
    }
    s = (s + 1) & mask;
  }
  // one counter update per warp for the slots its lanes claimed
  const uint32_t act = __activemask(), ball = __ballot_sync(act, won);
  const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
  uint32_t base = 0;
  if (lane == leader && ball) base = atomicAdd(n_rec, (uint32_t)__popc(ball));
  base = __shfl_sync(act, base, leader);
  if (won) {
    const uint32_t r = base + __popc(ball & ((1u << lane) - 1));
    if (key_form(r + 1, n) != KGV_KEYS_INLINE) {  // (r < the host's bound of the rec_rep / record arrays)
      rec_rep[r] = (uint32_t)i;
      table[s].rec = r + 1;
    }
  }
  item_slot[i] = s;
}

// One thread per record: the key's verdict, and for a good key P and its joint table (key_joint_record_build) or its odd-multiples table and zs (key_rec_build).
// It uses no shared memory, so its occupancy is its own (unbounded, ptxas takes 255 registers and two blocks per SM).  Five blocks per SM
// (96 registers, 84 480 resident threads: the bench shape's 70 794 records in one wave) measured 2.24 ms at the bench shape against
// 2.43 ms at three blocks (168 registers, 1.4 waves) and 2.46 ms at four, despite the larger spill code (DESIGN.md §4 K1).
#ifndef KGV_PREP_BLOCKS_PER_SM
#define KGV_PREP_BLOCKS_PER_SM 5
#endif
template <bool ECDSA>
__global__ void __launch_bounds__(KGV_BLOCK, KGV_PREP_BLOCKS_PER_SM) k_key_prepare(const uint8_t* __restrict__ pk, size_t n_arg, const uint32_t* __restrict__ n_dev,
                                                                              const uint32_t* __restrict__ rec_rep, const uint32_t* __restrict__ n_rec,
                                                                              uint32_t* __restrict__ recs) {
  const size_t n = n_dev ? (size_t)*n_dev : n_arg;
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  const int f = key_form(*n_rec, n);
  if (r >= *n_rec || f == KGV_KEYS_INLINE) return;
  uint32_t w[9];
  key_words<false, ECDSA>(w, pk, rec_rep[r]);
  if (f == KGV_KEYS_COMB) key_joint_record_build(recs + (size_t)r * KGV_JR_WORDS, ECDSA ? w[8] : 2u, w);
  else key_rec_build(recs + (size_t)r * KGV_KR_WORDS, ECDSA ? w[8] : 2u, w);
}

// Each thread verifies KGV_ITEMS consecutive-stride items (i = tid + j * total_threads: coalesced) and shares
// ONE modular inversion among them (Montgomery's trick): the field inversion of BIP-340's final affine
// conversion, resp. the scalar inversion s^-1 of ECDSA, drops from 1 to 1/KGV_ITEMS per signature with no
// cross-thread synchronisation.  Pending state sits in (L1-resident) local memory between the phases.
// The product of the trick: in the field for Schnorr, mod n for ECDSA.
template <bool ECDSA>
__device__ __forceinline__ void batch_mul(fe& r, const fe& a, const fe& b) {
  if constexpr (ECDSA) sc_mul(r.v, a.v, b.v);
  else fe_mul(r, a, b);
}
// The body of both verify kernels.  INDEXED: verify only the listed items (the signature-cache misses), their count read on the device.
// A separate instantiation: the two extra pointers live across the whole kernel cost the plain form 3 % (register pressure at the
// 168-register cap, measured).
template <bool ECDSA, bool ALIGNED, bool INDEXED>
__device__ __forceinline__ void verify_body(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig,
                                            size_t n_arg, uint8_t* __restrict__ status, const uint32_t* __restrict__ gtab,
                                            const uint32_t* __restrict__ index, const uint32_t* __restrict__ n_dev, KeyCacheView kc) {
  extern __shared__ uint32_t smem[];
  const size_t n = (INDEXED && n_dev) ? (size_t)*n_dev : n_arg;
  const size_t total = (size_t)gridDim.x * KGV_BLOCK;
  const size_t tid = (size_t)blockIdx.x * KGV_BLOCK + threadIdx.x;
  SmemTab tab{smem + threadIdx.x};
  // pending items: D, the value to invert (Schnorr: the true Z of R; ECDSA: s), and pre, the product of the earlier items' D;
  // X, Y: R before its affine conversion (Schnorr) or the key (ECDSA, inline key path); RX: r.  M, KR: ECDSA's m and key record, and
  // comb its form, the same for every item of a launch (a flag per item cost 32 B of stack)
  fe X[KGV_ITEMS], Y[KGV_ITEMS], RX[KGV_ITEMS], D[KGV_ITEMS], pre[KGV_ITEMS], M[KGV_ITEMS];
  const uint32_t* KR[KGV_ITEMS];
  bool comb = false;
  uint8_t st[KGV_ITEMS];
  // persistent grid (one resident wave): every thread walks the batch with stride total*KGV_ITEMS, so all
  // SM slots finish within one item of each other whatever n is (no wave quantisation)
#pragma unroll 1
  for (size_t base = 0; base < n; base += total * KGV_ITEMS) {
  fe acc;
  fe_set_u32(acc, 1);
  bool any = false;
#pragma unroll 1
  for (int j = 0; j < KGV_ITEMS; j++) {
    size_t i = base + tid + (size_t)j * total;
    st[j] = KGV_ST_INVALID;
    if (i >= n) continue;
    if (INDEXED) i = index[i];
    uint32_t pkw[9], mw[8], sw[16];
    key_words<ALIGNED, ECDSA>(pkw, pk, i);
    load_be32<ALIGNED>(mw, msg + 32 * i);
    load_be32<ALIGNED>(sw, sig + 64 * i);
    load_be32<ALIGNED>(sw + 8, sig + 64 * i + 32);
    const KeySrc key = kc.key_of(i, n);
    fe x, y, rx, d, m;
    uint8_t s1;
    if constexpr (ECDSA) s1 = ecdsa_phase1(x, y, rx.v, d.v, m.v, pkw[8], pkw, mw, sw, key);
    else s1 = schnorr_phase1(x, y, d, rx, pkw, mw, sw, tab, gtab, GLoadDev(), key);
    st[j] = s1;
    if (s1 == KGV_ST_PENDING) {
      X[j] = x; Y[j] = y; RX[j] = rx; D[j] = d;
      if constexpr (ECDSA) { M[j] = m; KR[j] = key.rec; comb = key.comb; }
      pre[j] = acc;
      batch_mul<ECDSA>(acc, acc, d);
      any = true;
    }
  }
  if (any) {
    fe inv;
    if constexpr (ECDSA) sc_inv(inv.v, acc.v);
    else fe_inv(inv, acc);
#pragma unroll 1
    for (int j = KGV_ITEMS - 1; j >= 0; j--) {
      if (st[j] != KGV_ST_PENDING) continue;
      fe di;  // 1 / D[j]
      batch_mul<ECDSA>(di, inv, pre[j]);
      batch_mul<ECDSA>(inv, inv, D[j]);
      if constexpr (ECDSA) st[j] = ecdsa_phase2(X[j], Y[j], RX[j].v, di.v, M[j].v, tab, gtab, GLoadDev(), KeySrc{KR[j], comb});
      else st[j] = schnorr_phase2(X[j], Y[j], di, RX[j]);
    }
  }
#pragma unroll 1
  for (int j = 0; j < KGV_ITEMS; j++) {
    size_t i = base + tid + (size_t)j * total;
    if (i < n) status[INDEXED ? index[i] : i] = st[j];
  }
  }
}

template <bool ALIGNED, bool INDEXED>
__global__ void __launch_bounds__(KGV_BLOCK, KGV_BLOCKS_PER_SM)
k_schnorr_verify(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig, size_t n_arg,
                 uint8_t* __restrict__ status, const uint32_t* __restrict__ gtab, const uint32_t* __restrict__ index, const uint32_t* __restrict__ n_dev,
                 KeyCacheView kc) {
  verify_body<false, ALIGNED, INDEXED>(pk, msg, sig, n_arg, status, gtab, index, n_dev, kc);
}
template <bool ALIGNED, bool INDEXED>
__global__ void __launch_bounds__(KGV_BLOCK, KGV_BLOCKS_PER_SM)
k_ecdsa_verify(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig, size_t n_arg,
               uint8_t* __restrict__ status, const uint32_t* __restrict__ gtab, const uint32_t* __restrict__ index, const uint32_t* __restrict__ n_dev,
               KeyCacheView kc) {
  verify_body<true, ALIGNED, INDEXED>(pk, msg, sig, n_arg, status, gtab, index, n_dev, kc);
}
using VerifyKernel = void (*)(const uint8_t*, const uint8_t*, const uint8_t*, size_t, uint8_t*, const uint32_t*, const uint32_t*, const uint32_t*,
                              KeyCacheView);
// every verify instantiation, [ecdsa][indexed][aligned]
static const VerifyKernel k_verify[2][2][2] = {
    {{k_schnorr_verify<false, false>, k_schnorr_verify<true, false>}, {k_schnorr_verify<false, true>, k_schnorr_verify<true, true>}},
    {{k_ecdsa_verify<false, false>, k_ecdsa_verify<true, false>}, {k_ecdsa_verify<false, true>, k_ecdsa_verify<true, true>}}};

// audit/debug: one signature, every traced intermediate written to dbg[stage*16 ..]
struct DevTrace {
  uint32_t* out;
  __device__ __forceinline__ void operator()(int stage, const uint32_t* w, int n) const {
    for (int i = 0; i < n && i < 16; i++) out[stage * 16 + i] = w[i];
  }
};
__global__ void __launch_bounds__(KGV_BLOCK, KGV_BLOCKS_PER_SM)
k_schnorr_trace(const uint8_t* __restrict__ pk, const uint8_t* __restrict__ msg, const uint8_t* __restrict__ sig,
                uint8_t* __restrict__ status, const uint32_t* __restrict__ gtab, uint32_t* __restrict__ dbg) {
  extern __shared__ uint32_t smem[];
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t pkw[8], mw[8], sw[16];
  load_be32<false>(pkw, pk);
  load_be32<false>(mw, msg);
  load_be32<false>(sw, sig);
  load_be32<false>(sw + 8, sig + 32);
  SmemTab tab{smem + threadIdx.x};
  status[0] = schnorr_verify_core(pkw, mw, sw, tab, gtab, GLoadDev(), DevTrace{dbg});
}

// audit/debug: exercise the arithmetic primitives directly (PTX bodies) on caller-provided operands.
// in: n items x 16 words (a[8], b[8]); out: n items x 16 words.
__global__ void k_selftest(int op, const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t a[8], b[8], r[16];
#pragma unroll
  for (int k = 0; k < 8; k++) { a[k] = in[i * 16 + k]; b[k] = in[i * 16 + 8 + k]; }
#pragma unroll
  for (int k = 0; k < 16; k++) r[k] = 0;
  fe fa, fb, fr;
#pragma unroll
  for (int k = 0; k < 8; k++) { fa.v[k] = a[k]; fb.v[k] = b[k]; }
  switch (op) {
    case 0: mul_wide(r, a, b); break;
    case 1: sqr_wide(r, a); break;
    case 2: fe_mul(fr, fa, fb); for (int k = 0; k < 8; k++) r[k] = fr.v[k]; break;
    case 3: fe_sqr(fr, fa); for (int k = 0; k < 8; k++) r[k] = fr.v[k]; break;
    case 4: sc_mul(r, a, b); break;
    case 5: sc_sqr(r, a); break;
    case 6: sc_inv(r, a); break;
    case 7: fe_inv(fr, fa); for (int k = 0; k < 8; k++) r[k] = fr.v[k]; break;
    case 8: fe_add(fr, fa, fb); for (int k = 0; k < 8; k++) r[k] = fr.v[k]; break;
    case 9: fe_sub(fr, fa, fb); for (int k = 0; k < 8; k++) r[k] = fr.v[k]; break;
    case 10: { uint32_t t[16]; mul_wide(t, a, b); sc_reduce512(r, t); } break;
    case 11: { uint32_t k1[5], k2[5]; bool n1, n2; glv_split(k1, n1, k2, n2, a); for (int k = 0; k < 5; k++) { r[k] = k1[k]; r[8 + k] = k2[k]; } r[5] = n1; r[13] = n2; } break;
    default: break;
  }
#pragma unroll
  for (int k = 0; k < 16; k++) out[i * 16 + k] = r[k];
}

// audit/debug: the eight-lane field primitives (kgv_lanes.cuh), one item per group of eight lanes, same in/out layout
// as k_selftest.  A group past n leaves as a whole group (n * 8 threads, groups never straddle the bound).
__global__ void k_selftest_lanes(int op, const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n) {
  const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 3);
  if (i >= n) return;
  const lane_grp g = lane_group();
  const uint32_t a = in[i * 16 + g.k], b = in[i * 16 + 8 + g.k];
  uint32_t r = 0;
  switch (op) {
    case 12: r = fe_mul_lanes(a, b, g); break;
    case 13: r = fe_sqr_lanes(a, g); break;
    default: break;
  }
  out[i * 16 + g.k] = r;
  out[i * 16 + 8 + g.k] = 0;
}

__global__ void k_status_to_bitmap(const uint8_t* __restrict__ status, size_t n, uint8_t* __restrict__ bitmap) {
  size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t nbytes = (n + 7) / 8;
  if (b >= nbytes) return;
  uint32_t bits = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    size_t i = 8 * b + j;
    if (i < n && status[i] == KGV_ST_VALID) bits |= 1u << j;
  }
  bitmap[b] = (uint8_t)bits;
}

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
// 1 = device-accessible pointer, 0 = host pointer
int kgv_ptr_is_device(const void* p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

int kgv_host_only(kgv_ctx* ctx, const char* call, const char* what, const void* p) {
  if (!p || !kgv_ptr_is_device(p)) return KGV_OK;
  ctx->err = std::string(call) + ": " + what + " must be host memory";
  return KGV_ERR_ARG;
}

bool kgv_io::is_device(const void* p) {
  for (int i = 0; i < n_side; i++)
    if (side[i].p == p) return side[i].dev;
  const bool dev = kgv_ptr_is_device(p) != 0;
  if (n_side < 16) side[n_side++] = {p, dev};
  return dev;
}

int kgv_io::one_side(const char* call, std::initializer_list<const void*> ps, bool* dev) {
  int first = -1;  // side of the first non-null pointer
  for (const void* p : ps) {
    if (!p) continue;
    const int d = is_device(p);
    if (first < 0) first = d;
    else if (d != first) {
      ctx->err = std::string(call) + ": the arrays of one call must be all host pointers or all device pointers";
      return KGV_ERR_ARG;
    }
  }
  if (dev) *dev = first == 1;
  return KGV_OK;
}

void kgv_io::add(const void* p, size_t bytes, const void** d, bool in, bool out) {
  *d = p;
  if (!p || is_device(p)) return;
  arr[n_arr++] = {p, bytes, d, in, out};
  host_out |= out;
}

int kgv_io::stage() {
  size_t total = 0;
  for (int i = 0; i < n_arr; i++) total += al256(arr[i].bytes);
  if (total == 0) return KGV_OK;
  int rc = kgv_reserve(ctx, &ctx->d_io, &ctx->d_io_cap, total);
  if (rc) return rc;
  size_t o = 0;
  for (int i = 0; i < n_arr; i++) {
    *arr[i].d = ctx->d_io + o;
    if (arr[i].in && arr[i].bytes) CK(cudaMemcpyAsync(ctx->d_io + o, arr[i].p, arr[i].bytes, cudaMemcpyHostToDevice, ctx->stream));
    o += al256(arr[i].bytes);
  }
  return KGV_OK;
}

int kgv_io::copy_out(void* p, const void* d, size_t bytes) {
  const bool dev = is_device(p);
  host_out |= !dev;
  CK(cudaMemcpyAsync(p, d, bytes, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, ctx->stream));
  return KGV_OK;
}

void kgv_io::trim(const void* p, size_t bytes) {
  for (int i = 0; i < n_arr; i++)
    if (arr[i].p == p && bytes < arr[i].bytes) arr[i].bytes = bytes;
}

int kgv_io::finish() {
  for (int i = 0; i < n_arr; i++)
    if (arr[i].out && arr[i].bytes) CK(cudaMemcpyAsync((void*)arr[i].p, *arr[i].d, arr[i].bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (host_out) CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}

// Per-call device buffers only ever grow.  The outgrown allocation is NOT freed on the spot: cudaFree synchronises the whole device, which
// stalls every other stream and deadlocks a process that drives several contexts of one device whose kernels wait for each other (the
// peer-exchange wait kernels of kgv_comm.cu); cudaMallocAsync was tried and blocks in the same situation (measured).  Outgrown buffers are
// parked and released by kgv_synchronize / kgv_destroy, i.e. at points where the caller has declared the context idle.  Growth is
// geometric (x1.25), so the parked memory stays below ~4x the live buffer.
int kgv_malloc(kgv_ctx* ctx, void** p, size_t bytes) {
  cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) {
    // memory pressure: now it is worth a device synchronisation to give the parked buffers back and try again
    (void)cudaGetLastError();
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->aux_stream);
    for (uint8_t* q : ctx->parked) cudaFree(q);
    ctx->parked.clear();
    e = cudaMalloc(p, bytes);
  }
  if (e != cudaSuccess) { ctx->err = std::string("cudaMalloc failed: ") + cudaGetErrorString(e); (void)cudaGetLastError(); *p = nullptr; return KGV_ERR_NOMEM; }
  return KGV_OK;
}

int kgv_reserve(kgv_ctx* ctx, uint8_t** buf, size_t* cap, size_t need) {
  if (*cap >= need) return KGV_OK;
  if (*buf) { ctx->parked.push_back(*buf); *buf = nullptr; *cap = 0; }
  size_t want = need + need / 4 + 4096;
  int rc = kgv_malloc(ctx, (void**)buf, want);
  if (rc) return rc;
  *cap = want;
  return KGV_OK;
}

extern "C" int kgv_create(int device, uint32_t flags, kgv_ctx** out) {
  (void)flags;
  if (!out) return KGV_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    (void)cudaGetLastError();
    return KGV_ERR_CUDA;  // no CUDA device: there is no CPU path
  }
  kgv_ctx* ctx = new kgv_ctx();
  ctx->device = device;
  auto body = [&]() -> int {
    CK(cudaSetDevice(device));
    CK(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    CK(cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
    CK(cudaMalloc((void**)&ctx->gtab, (size_t)8 * 65536 * 16 * sizeof(uint32_t)));
    k_build_gtab<<<(8 * 65536) / 128, 128, 0, ctx->stream>>>(ctx->gtab);
    CK(cudaGetLastError());
    ctx->launches++;
    const int smem = KGV_BLOCK * 128 * (int)sizeof(uint32_t);
    for (const auto& kind : k_verify)
      for (const auto& form : kind)
        for (VerifyKernel k : form) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int per_sm = 0, sms = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_verify[0][0][1], KGV_BLOCK, smem));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    ctx->resident_blocks = per_sm * sms > 0 ? per_sm * sms : 132 * KGV_BLOCKS_PER_SM;  // 132 SMs: H100 SXM
    CK(cudaStreamSynchronize(ctx->stream));
    return KGV_OK;
  };
  int rc = body();
  if (rc != KGV_OK) {
    fprintf(stderr, "kgv_create: %s\n", ctx->err.c_str());
    delete ctx;
    return rc;
  }
  *out = ctx;
  return KGV_OK;
}

extern "C" void kgv_destroy(kgv_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (auto& P : ctx->prefetch) if (P.worker.joinable()) P.worker.join();
  if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->gtab) cudaFree(ctx->gtab);
  for (uint8_t* b : {ctx->d_io, ctx->d_in, ctx->d_out, ctx->d_batch, ctx->prefetch[0].buf, ctx->prefetch[1].buf, ctx->d_scratch, ctx->d_mu, ctx->d_work, ctx->d_replay, ctx->d_keys[0], ctx->d_keys[1]})
    if (b) cudaFree(b);
  for (uint8_t* b : ctx->parked) cudaFree(b);
  for (cudaEvent_t e : ctx->ev_chunk) if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->ev_time) if (e) cudaEventDestroy(e);
  if (ctx->ev_prefetch) cudaEventDestroy(ctx->ev_prefetch);
  for (auto& P : ctx->prefetch) if (P.done) cudaEventDestroy(P.done);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

extern "C" int kgv_set_stream(kgv_ctx* ctx, void* cuda_stream) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  ctx->stream = (cudaStream_t)cuda_stream;  // NULL is CUDA's default stream, exactly as in cudaStream_t
  return KGV_OK;
}

extern "C" int kgv_reset_stream(kgv_ctx* ctx) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  ctx->stream = ctx->own_stream;
  return KGV_OK;
}

extern "C" int kgv_synchronize(kgv_ctx* ctx) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (!ctx->parked.empty()) {  // the caller declared the context idle: outgrown buffers can go
    CK(cudaStreamSynchronize(ctx->aux_stream));
    if (ctx->copy_stream) CK(cudaStreamSynchronize(ctx->copy_stream));
    for (uint8_t* p : ctx->parked) cudaFree(p);
    ctx->parked.clear();
  }
  return KGV_OK;
}

extern "C" const char* kgv_last_error(const kgv_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
extern "C" uint64_t kgv_launch_count(const kgv_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---------------------------------------------------------------------------------------------
// signature verification entry points
// ---------------------------------------------------------------------------------------------
// Enqueues the per-launch key cache of a verify launch on st: table cleared, k_key_dedup, k_key_prepare.  Sized from the host's n (an
// upper bound of *n_dev when given); the scratch belongs to the item kind (Schnorr and ECDSA launches of one validation call run
// side by side on two streams) and lives until the next launch of that kind, which the stream order puts after this one.
static int key_cache_launch(kgv_ctx* ctx, const uint8_t* dpk, size_t n, bool ecdsa, bool aligned, cudaStream_t st, const uint32_t* index,
                            const uint32_t* n_dev, KeyCacheView* kc) {
  uint32_t slots = 64;
  while (slots < 2 * n) slots <<= 1;                       // load factor <= 1/2
  const uint32_t cap = (uint32_t)(n / 2 < KGV_KEY_RECORDS_MAX ? n / 2 : KGV_KEY_RECORDS_MAX);  // key_form's bounds
  const size_t cap_comb = n / KGV_COMB_USES < KGV_KEY_RECORDS_MAX ? n / KGV_COMB_USES : KGV_KEY_RECORDS_MAX;
  const size_t rec_bytes = std::max((size_t)cap * KGV_KR_WORDS, cap_comb * KGV_JR_WORDS) * 4;
  const size_t o_tab = 256, o_item = o_tab + (size_t)slots * sizeof(KeySlot);
  const size_t o_rep = (o_item + n * 4 + 255) & ~(size_t)255, o_rec = (o_rep + (size_t)cap * 4 + 255) & ~(size_t)255;
  int rc = kgv_reserve(ctx, &ctx->d_keys[ecdsa], &ctx->d_keys_cap[ecdsa], o_rec + rec_bytes);
  if (rc) return rc;
  uint8_t* K = ctx->d_keys[ecdsa];
  uint32_t* n_rec = (uint32_t*)K;
  KeySlot* table = (KeySlot*)(K + o_tab);
  uint32_t *item_slot = (uint32_t*)(K + o_item), *rec_rep = (uint32_t*)(K + o_rep), *recs = (uint32_t*)(K + o_rec);
  CK(cudaMemsetAsync(K, 0, o_item, st));
  const unsigned gd = (unsigned)((n + 255) / 256);
  // (ECDSA keys, at a 33-byte stride, are never word aligned)
  const auto dedup = ecdsa ? k_key_dedup<false, true> : aligned ? k_key_dedup<true, false> : k_key_dedup<false, false>;
  dedup<<<gd, 256, 0, st>>>(dpk, n, index, n_dev, table, slots - 1, item_slot, rec_rep, n_rec);
  CK(cudaGetLastError());
  ctx->launches++;
  if (cap) {
    const unsigned gp = (cap + KGV_BLOCK - 1) / KGV_BLOCK;
    const auto prepare = ecdsa ? k_key_prepare<true> : k_key_prepare<false>;
    prepare<<<gp, KGV_BLOCK, 0, st>>>(dpk, n, n_dev, rec_rep, n_rec, recs);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  *kc = KeyCacheView{table, item_slot, recs, n_rec};
  return KGV_OK;
}

int kgv_launch_verify(kgv_ctx* ctx, const uint8_t* dpk, const uint8_t* dmsg, const uint8_t* dsig, size_t n, uint8_t* dst, bool ecdsa,
                      cudaStream_t st, const uint32_t* index, const uint32_t* n_dev) {
  if (n == 0) return KGV_OK;
  if (n >= 0x7FFFFFFFu) return fail_arg(ctx, "verify launch of 2^31 or more items");
  const int smem = KGV_BLOCK * 128 * (int)sizeof(uint32_t);
  // one resident wave, persistent; items are strided by the grid size, so a batch smaller than the wave still
  // spreads over every SM (one item per thread) instead of packing KGV_ITEMS items into a quarter of the threads
  size_t want = (n + KGV_BLOCK - 1) / KGV_BLOCK;
  unsigned blocks = (unsigned)(want < (size_t)ctx->resident_blocks ? want : (size_t)ctx->resident_blocks);
  bool aligned = (((uintptr_t)dmsg | (uintptr_t)dsig | (ecdsa ? 0 : (uintptr_t)dpk)) & 31) == 0;
  // The key cache pays off when threads verify several items: in a launch of at most one item per thread the preparation's latency
  // comes on top of a verify that shortens by the same latency (small batches measured 10 % slower with it).
  KeyCacheView kc{};
  const bool key_cache = n > (size_t)ctx->resident_blocks * KGV_BLOCK;
  if (key_cache) {
    int rc = key_cache_launch(ctx, dpk, n, ecdsa, aligned, st, index, n_dev, &kc);
    if (rc) return rc;
  }
  if (!index) {
    auto& lv = ctx->last_verify[ecdsa];
    lv.n = n; lv.blocks = blocks; lv.key_cache = key_cache; lv.stream = st;
  }
  k_verify[ecdsa][index != nullptr][aligned]<<<blocks, KGV_BLOCK, smem, st>>>(dpk, dmsg, dsig, n, dst, ctx->gtab, index, n_dev, kc);
  CK(cudaGetLastError());
  ctx->launches++;
  return KGV_OK;
}

static int verify_common(kgv_ctx* ctx, const uint8_t* pk, size_t pk_stride, const uint8_t* msg, const uint8_t* sig, size_t n,
                         uint8_t* status, bool ecdsa) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!pk || !msg || !sig || !status) return fail_arg(ctx, "null buffer");
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  bool dev;
  if (int rc = io.one_side(ecdsa ? "kgv_ecdsa_verify" : "kgv_schnorr_verify", {pk, msg, sig, status}, &dev)) return rc;
  // Large host batches are uploaded in chunks of one full persistent wave (resident threads x KGV_ITEMS signatures) on the
  // side stream while the previous chunk is being verified: only the first chunk's upload is exposed.
  const size_t chunk = (size_t)ctx->resident_blocks * KGV_BLOCK * KGV_ITEMS;
  if (!dev && n >= 2 * chunk && (n + chunk - 1) / chunk <= 32) {
    size_t off_msg = (pk_stride * n + 255) & ~(size_t)255;
    size_t off_sig = off_msg + 32 * n;
    int rc = kgv_reserve(ctx, &ctx->d_in, &ctx->d_in_cap, off_sig + 64 * n);
    if (rc) return rc;
    rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, n);
    if (rc) return rc;
    const uint8_t *dpk = ctx->d_in, *dmsg = ctx->d_in + off_msg, *dsig = ctx->d_in + off_sig;
    uint8_t* dst = ctx->d_out;
    CK(cudaEventRecord(ctx->ev_fork, ctx->stream));          // the staging buffers may still be read by earlier work of this stream
    CK(cudaStreamWaitEvent(ctx->aux_stream, ctx->ev_fork, 0));
    size_t c = 0;
    for (size_t a = 0; a < n; a += chunk, c++) {
      const size_t m = n - a < chunk ? n - a : chunk;
      if (!ctx->ev_chunk[c]) CK(cudaEventCreateWithFlags(&ctx->ev_chunk[c], cudaEventDisableTiming));
      CK(cudaMemcpyAsync(ctx->d_in + pk_stride * a, pk + pk_stride * a, pk_stride * m, cudaMemcpyHostToDevice, ctx->aux_stream));
      CK(cudaMemcpyAsync(ctx->d_in + off_msg + 32 * a, msg + 32 * a, 32 * m, cudaMemcpyHostToDevice, ctx->aux_stream));
      CK(cudaMemcpyAsync(ctx->d_in + off_sig + 64 * a, sig + 64 * a, 64 * m, cudaMemcpyHostToDevice, ctx->aux_stream));
      CK(cudaEventRecord(ctx->ev_chunk[c], ctx->aux_stream));
      CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_chunk[c], 0));
      int rc2 = kgv_launch_verify(ctx, dpk + pk_stride * a, dmsg + 32 * a, dsig + 64 * a, m, dst + a, ecdsa, ctx->stream);
      if (rc2) return rc2;
    }
    if ((rc = io.copy_out(status, dst, n))) return rc;
    return io.finish();
  }
  const uint8_t *dpk, *dmsg, *dsig;
  uint8_t* dst;
  io.in(pk, pk_stride * n, &dpk);
  io.in(msg, 32 * n, &dmsg);
  io.in(sig, 64 * n, &dsig);
  io.out(status, n, &dst);
  if (int rc = io.stage()) return rc;
  if (int rc = kgv_launch_verify(ctx, dpk, dmsg, dsig, n, dst, ecdsa, ctx->stream)) return rc;
  return io.finish();
}

extern "C" int kgv_schnorr_verify(kgv_ctx* ctx, const uint8_t* pk32, const uint8_t* msg32, const uint8_t* sig64, size_t n, uint8_t* status) {
  return verify_common(ctx, pk32, 32, msg32, sig64, n, status, false);
}
extern "C" int kgv_ecdsa_verify(kgv_ctx* ctx, const uint8_t* pk33, const uint8_t* msg32, const uint8_t* sig64, size_t n, uint8_t* status) {
  return verify_common(ctx, pk33, 33, msg32, sig64, n, status, true);
}

extern "C" int kgv_status_to_bitmap(kgv_ctx* ctx, const uint8_t* status, size_t n, uint8_t* bitmap) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (n == 0) return KGV_OK;
  if (!status || !bitmap) return fail_arg(ctx, "null buffer");
  CK(cudaSetDevice(ctx->device));
  kgv_io io(ctx);
  if (int rc = io.one_side("kgv_status_to_bitmap", {status, bitmap})) return rc;
  size_t nbytes = (n + 7) / 8;
  const uint8_t* dsrc;
  uint8_t* ddst;
  io.in(status, n, &dsrc);
  io.out(bitmap, nbytes, &ddst);
  if (int rc = io.stage()) return rc;
  k_status_to_bitmap<<<(unsigned)((nbytes + 255) / 256), 256, 0, ctx->stream>>>(dsrc, n, ddst);
  CK(cudaGetLastError());
  ctx->launches++;
  return io.finish();
}

extern "C" int kgv_debug_schnorr_trace(kgv_ctx* ctx, const uint8_t* pk32, const uint8_t* msg32, const uint8_t* sig64, uint32_t* trace_words,
                                       uint8_t* status) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!pk32 || !msg32 || !sig64 || !trace_words || !status) return fail_arg(ctx, "null buffer");
  CK(cudaSetDevice(ctx->device));
  const size_t tw = KGV_TRACE_STAGES * 16 * sizeof(uint32_t);
  int rc = kgv_reserve(ctx, &ctx->d_in, &ctx->d_in_cap, 256);
  if (rc) return rc;
  rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, tw + 256);
  if (rc) return rc;
  CK(cudaMemcpyAsync(ctx->d_in, pk32, 32, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_in + 32, msg32, 32, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->d_in + 64, sig64, 64, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_out, 0, tw + 256, ctx->stream));
  const int smem = KGV_BLOCK * 128 * (int)sizeof(uint32_t);
  CK(cudaFuncSetAttribute(k_schnorr_trace, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_schnorr_trace<<<1, KGV_BLOCK, smem, ctx->stream>>>(ctx->d_in, ctx->d_in + 32, ctx->d_in + 64, ctx->d_out + tw, ctx->gtab, (uint32_t*)ctx->d_out);
  CK(cudaGetLastError());
  ctx->launches++;
  CK(cudaMemcpyAsync(trace_words, ctx->d_out, tw, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(status, ctx->d_out + tw, 1, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}

extern "C" int kgv_debug_key_form(kgv_ctx* ctx, int ecdsa, kgv_key_form_info* out) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!out) return fail_arg(ctx, "null buffer");
  const auto& lv = ctx->last_verify[ecdsa ? 1 : 0];
  if (lv.n == 0) return fail_arg(ctx, "no verify launch of that kind yet");
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(lv.stream));
  uint32_t n_rec = 0;
  if (lv.key_cache) CK(cudaMemcpy(&n_rec, ctx->d_keys[ecdsa ? 1 : 0], sizeof n_rec, cudaMemcpyDeviceToHost));
  out->n_items = lv.n;
  out->threads = (uint64_t)lv.blocks * KGV_BLOCK;
  out->distinct_keys = n_rec;
  if (!lv.key_cache) out->form = KGV_KEY_FORM_NO_CACHE;
  else {
    const int f = key_form(n_rec, lv.n);
    out->form = f == KGV_KEYS_COMB ? KGV_KEY_FORM_COMB : f == KGV_KEYS_PLAIN ? KGV_KEY_FORM_PLAIN : KGV_KEY_FORM_INLINE;
  }
  return KGV_OK;
}

extern "C" int kgv_debug_selftest(kgv_ctx* ctx, int op, const uint32_t* in_words, uint32_t* out_words, size_t n) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!in_words || !out_words || n == 0 || n > (1u << 20)) return fail_arg(ctx, "bad selftest arguments");
  CK(cudaSetDevice(ctx->device));
  int rc = kgv_reserve(ctx, &ctx->d_in, &ctx->d_in_cap, n * 64);
  if (rc) return rc;
  rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, n * 64);
  if (rc) return rc;
  CK(cudaMemcpyAsync(ctx->d_in, in_words, n * 64, cudaMemcpyHostToDevice, ctx->stream));
  if (op >= 12)
    k_selftest_lanes<<<(unsigned)((n * 8 + 63) / 64), 64, 0, ctx->stream>>>(op, (const uint32_t*)ctx->d_in, (uint32_t*)ctx->d_out, (int)n);
  else
    k_selftest<<<(unsigned)((n + 63) / 64), 64, 0, ctx->stream>>>(op, (const uint32_t*)ctx->d_in, (uint32_t*)ctx->d_out, (int)n);
  CK(cudaGetLastError());
  ctx->launches++;
  CK(cudaMemcpyAsync(out_words, ctx->d_out, n * 64, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}

extern "C" int kgv_gtable_entry(kgv_ctx* ctx, int which, uint32_t v, uint8_t out_xy[64]) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if ((which != 0 && which != 1) || v == 0 || v > 65535 || !out_xy) return fail_arg(ctx, "bad table index");
  CK(cudaSetDevice(ctx->device));
  uint32_t w[16];
  CK(cudaMemcpyAsync(w, ctx->gtab + ((size_t)which * 4 * 65536 + v) * 16, sizeof w, cudaMemcpyDeviceToHost, ctx->stream));  // v*G, v*2^128*G
  CK(cudaStreamSynchronize(ctx->stream));
  for (int c = 0; c < 2; c++)
    for (int i = 0; i < 8; i++) {
      uint32_t limb = w[c * 8 + 7 - i];
      out_xy[c * 32 + 4 * i] = (uint8_t)(limb >> 24);
      out_xy[c * 32 + 4 * i + 1] = (uint8_t)(limb >> 16);
      out_xy[c * 32 + 4 * i + 2] = (uint8_t)(limb >> 8);
      out_xy[c * 32 + 4 * i + 3] = (uint8_t)limb;
    }
  return KGV_OK;
}
