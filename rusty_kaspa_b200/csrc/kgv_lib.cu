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
  const uint32_t* item_rec;   // a launch over stored keys only (kgv_keycache): item -> its stored comb record + 1; nullptr: not such a launch
  const uint32_t* kc_recs;    // that cache's records, KGV_JR_WORDS words each
  // the key source of item i: its stored record, else its record and the launch's form, or no record (the launch makes none)
  __device__ __forceinline__ KeySrc key_of(size_t i, size_t n) const {
    if (item_rec) return KeySrc{kc_recs + (size_t)(item_rec[i] - 1) * KGV_JR_WORDS, true};
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
// the remaining items stop (the verify kernels then take the inline key path for every item).  ALL: every distinct key gets a
// representative until there are more than `limit` (the device key cache's misses, kgv_keycache below).
template <bool ALIGNED, bool ECDSA, bool ALL = false>
__global__ void __launch_bounds__(256) k_key_dedup(const uint8_t* __restrict__ pk, size_t n_arg, const uint32_t* __restrict__ index,
                                                   const uint32_t* __restrict__ n_dev, KeySlot* __restrict__ table, uint32_t mask,
                                                   uint32_t* __restrict__ item_slot, uint32_t* __restrict__ rec_rep, uint32_t* n_rec,
                                                   uint32_t limit) {
  const size_t n = n_dev ? (size_t)*n_dev : n_arg;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  if (ALL ? *(volatile uint32_t*)n_rec > limit : key_form(*(volatile uint32_t*)n_rec, n) == KGV_KEYS_INLINE) return;
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
    if (ALL || key_form(r + 1, n) != KGV_KEYS_INLINE) {  // (r < the host's bound of the rec_rep / record arrays)
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

// ---- device key cache (kgv_keycache, include/kgv.h): comb-form key records kept across the verify launches of the contexts sharing it ----
// One partition per item kind.  Set-associative: a key's set is its key_hash modulo the number of sets; slot s of the partition owns
// record s (KGV_JR_WORDS words), so there is no allocator and a lookup reads one set.  stamp: the partition launch that last used the
// slot (0: empty).  A launch stamps the slots it reads, and an insert only takes a slot stamped by an earlier launch (the empty one first,
// then the least recently used), so no launch evicts a record it reads.
#define KGV_KC_WAYS 8
struct KcSet {
  uint32_t stamp[KGV_KC_WAYS];
  uint32_t fp[KGV_KC_WAYS];           // high half of the key's hash
  uint32_t key[KGV_KC_WAYS][9];       // key_words: x, and the tag for ECDSA
};
struct KcPart {
  KcSet* sets;
  uint32_t* recs;
  uint32_t n_sets;                     // 0: the kind has no partition
  unsigned long long* ctr;             // [0] lookups, [1] hits, [2] inserts, [3] evictions
};
// per-launch words of a partition's scratch
enum { KC_N = 0, KC_ORD_HIT = 1, KC_N_MISS = 2, KC_DIST_HIT = 3, KC_TAKE = 4, KC_N_REC = 5, KC_ORD_MISS = 6 };
enum { KC_COUNT = 1, KC_ORDER = 2, KC_GATED = 4 };

// position of this lane among the active lanes with pred, after the earlier warps' (one atomic per warp)
__device__ __forceinline__ uint32_t warp_claim(uint32_t* ctr, bool pred) {
  const uint32_t act = __activemask(), ball = __ballot_sync(act, pred);
  const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
  uint32_t base = 0;
  if (lane == leader && ball) base = atomicAdd(ctr, (uint32_t)__popc(ball));
  return __shfl_sync(act, base, leader) + __popc(ball & ((1u << lane) - 1));
}
__device__ __forceinline__ void warp_count(unsigned long long* ctr, bool pred) {
  const uint32_t act = __activemask(), ball = __ballot_sync(act, pred);
  if ((threadIdx.x & 31) == __ffs(act) - 1 && ball) atomicAdd(ctr, (unsigned long long)__popc(ball));
}

// One thread per item the launch verifies (index and n_dev honoured): probes the key's set.
//   KC_COUNT  counts lookups, stamps the hit slots (KC_DIST_HIT: distinct slots hit), and appends each miss's key bytes to miss_keys
//             (KC_N_MISS of them), the input of the insert
//   KC_ORDER  counts the hits (items the stored-record launch verifies); item_rec[i] = slot + 1 of a hit; the hits listed in order
//             (KC_ORD_HIT of them), the misses in miss_order (KC_ORD_MISS):
//             two verify launches, each of one key form.  (A block never mixes forms: ecmult_joint's staging and the inline path's
//             odd-multiples table lay the threads' shared memory out differently, so a thread of one form overwrites its neighbours'.)
//   KC_GATED  the launch's insert did not take it (KC_TAKE == 0): every item in miss_order, as given
template <bool ALIGNED, bool ECDSA>
__global__ void __launch_bounds__(256) k_kc_lookup(const uint8_t* __restrict__ pk, size_t n_arg, const uint32_t* __restrict__ index,
                                                   const uint32_t* __restrict__ n_dev, KcPart p, uint32_t stamp, int mode, uint32_t* hdr,
                                                   uint32_t* __restrict__ item_rec, uint32_t* __restrict__ order, uint32_t* __restrict__ miss_order,
                                                   uint8_t* __restrict__ miss_keys) {
  const size_t n = n_dev ? (size_t)*n_dev : n_arg;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0 && (mode & KC_COUNT)) hdr[KC_N] = (uint32_t)n;
  const bool taken = !(mode & KC_GATED) || *(volatile uint32_t*)(hdr + KC_TAKE);
  if (t == 0 && !taken) hdr[KC_ORD_MISS] = (uint32_t)n;
  if (t >= n) return;
  const size_t i = index ? index[t] : t;
  if (!taken) {
    miss_order[t] = (uint32_t)i;
    return;
  }
  const int nw = ECDSA ? 9 : 8;
  uint32_t w[9];
  key_words<ALIGNED, ECDSA>(w, pk, i);
  const uint64_t h = key_hash(w, nw);
  const uint32_t set = (uint32_t)(h % p.n_sets), fp = (uint32_t)(h >> 32);
  KcSet* s = p.sets + set;
  int way = -1;
  for (int k = 0; k < KGV_KC_WAYS && way < 0; k++) {
    if (!s->stamp[k] || s->fp[k] != fp) continue;
    bool eq = true;
    for (int q = 0; q < nw; q++) eq = eq && s->key[k][q] == w[q];
    if (eq) way = k;
  }
  const bool hit = way >= 0;
  if (mode & KC_COUNT) {
    if (hit && atomicExch(&s->stamp[way], stamp) != stamp) atomicAdd(&hdr[KC_DIST_HIT], 1u);
    const uint32_t k = warp_claim(&hdr[KC_N_MISS], !hit);
    if (!hit) {
      const int len = ECDSA ? 33 : 32;
      for (int b = 0; b < len; b++) miss_keys[(size_t)len * k + b] = pk[(size_t)len * i + b];
    }
    warp_count(&p.ctr[0], true);
  }
  if (mode & KC_ORDER) {
    warp_count(&p.ctr[1], hit);
    if (hit) item_rec[i] = set * KGV_KC_WAYS + way + 1;
    const uint32_t h_pos = warp_claim(&hdr[KC_ORD_HIT], hit), m_pos = warp_claim(&hdr[KC_ORD_MISS], !hit);
    if (hit) order[h_pos] = (uint32_t)i;
    else miss_order[m_pos] = (uint32_t)i;
  }
}

// One thread per distinct miss (k_key_dedup<.., true> over miss_keys): takes a slot of the key's set stamped by an earlier launch (empty
// first, then the least recently used), writes the key and builds its comb-form record there (key_joint_record_build).  A set whose every
// slot this launch uses keeps its records; the key is then not stored.  gate (launches of more items than resident threads): insert only
// when today's rule would make records for the launch's keys (key_form over the distinct hits and misses) or nothing is missing, and the
// partition holds them all; KC_TAKE = 1 then, and the verify reads every record from the partition.
template <bool ECDSA>
__global__ void __launch_bounds__(KGV_BLOCK, KGV_PREP_BLOCKS_PER_SM) k_kc_insert(KcPart p, const uint8_t* __restrict__ miss_keys,
                                                                            const uint32_t* __restrict__ rec_rep, uint32_t* hdr, uint32_t stamp, bool gate) {
  const uint32_t n_rec = hdr[KC_N_REC];
  if (gate) {
    const uint32_t keys = hdr[KC_DIST_HIT] + n_rec;
    const bool take = keys <= p.n_sets * KGV_KC_WAYS && (n_rec == 0 || key_form(keys, hdr[KC_N]) != KGV_KEYS_INLINE);
    if (!take) return;
    if (blockIdx.x == 0 && threadIdx.x == 0) hdr[KC_TAKE] = 1;
  }
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rec) return;
  const int nw = ECDSA ? 9 : 8;
  uint32_t w[9];
  key_words<false, ECDSA>(w, miss_keys, rec_rep[r]);
  const uint64_t h = key_hash(w, nw);
  const uint32_t set = (uint32_t)(h % p.n_sets);
  KcSet* s = p.sets + set;
  int way;
  uint32_t old;
  for (;;) {
    way = -1;
    old = stamp;
    for (int k = 0; k < KGV_KC_WAYS; k++) {
      const uint32_t v = *(volatile uint32_t*)&s->stamp[k];
      if (v < old) { old = v; way = k; }
    }
    if (way < 0) return;
    if (atomicCAS(&s->stamp[way], old, stamp) == old) break;
  }
  s->fp[way] = (uint32_t)(h >> 32);
  for (int q = 0; q < nw; q++) s->key[way][q] = w[q];
  atomicAdd(&p.ctr[2], 1ull);
  if (old) atomicAdd(&p.ctr[3], 1ull);
  key_joint_record_build(p.recs + (size_t)(set * KGV_KC_WAYS + way) * KGV_JR_WORDS, ECDSA ? w[8] : 2u, w);
}

// a launch the device key cache took makes no per-launch records: its n_rec is set past every bound, so k_key_dedup and k_key_prepare
// return at once and key_of finds no per-launch record
__global__ void k_kc_stand_down(const uint32_t* hdr, uint32_t* n_rec) {
  if (hdr[KC_TAKE]) *n_rec = 0xFFFFFFFFu;
}
// stamps wrap after 2^32 launches of a partition: every used slot restarts at 1
__global__ void k_kc_restamp(KcSet* sets, uint32_t n_sets) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sets) return;
  for (int k = 0; k < KGV_KC_WAYS; k++)
    if (sets[s].stamp[k]) sets[s].stamp[k] = 1;
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

static void keycache_quiesce(kgv_keycache* kc);
static void keycache_free(kgv_ctx* ctx);

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
    if (ctx->keycache) keycache_quiesce(ctx->keycache);  // a deferred key insert may still read a parked scratch
    for (uint8_t* q : ctx->parked) cudaFree(q);
    ctx->parked.clear();
    kgv_release_retired(ctx, false);
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
  keycache_free(ctx);
  if (ctx->gtab) cudaFree(ctx->gtab);
  for (uint8_t* b : {ctx->d_io, ctx->d_in, ctx->d_out, ctx->d_batch, ctx->prefetch[0].buf, ctx->prefetch[1].buf, ctx->d_scratch, ctx->d_mu, ctx->d_work, ctx->d_replay, ctx->d_keys[0], ctx->d_keys[1]})
    if (b) cudaFree(b);
  for (uint8_t* b : ctx->parked) cudaFree(b);
  kgv_release_retired(ctx, true);
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
    if (ctx->keycache) keycache_quiesce(ctx->keycache);
    for (uint8_t* p : ctx->parked) cudaFree(p);
    ctx->parked.clear();
  }
  kgv_release_retired(ctx, false);  // table arrays given up by this context's writes, once those writes have completed
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
// stand_down (may be null): the device key cache's launch words; when its insert took the launch, no per-launch record is made.
static int key_cache_launch(kgv_ctx* ctx, const uint8_t* dpk, size_t n, bool ecdsa, bool aligned, cudaStream_t st, const uint32_t* index,
                            const uint32_t* n_dev, KeyCacheView* kc, const uint32_t* stand_down = nullptr) {
  uint32_t slots = 64;
  while (slots < 2 * n) slots <<= 1;                       // load factor <= 1/2
  const uint32_t cap = (uint32_t)(n / 2 < KGV_KEY_RECORDS_MAX ? n / 2 : KGV_KEY_RECORDS_MAX);  // key_form's bounds
  const size_t cap_comb = n / KGV_COMB_USES < KGV_KEY_RECORDS_MAX ? n / KGV_COMB_USES : KGV_KEY_RECORDS_MAX;
  const size_t rec_words = std::max((size_t)cap * KGV_KR_WORDS, cap_comb * KGV_JR_WORDS);
  uint32_t *n_rec, *item_slot, *rec_rep, *recs;
  KeySlot* table;
  int rc = kgv_reserve_carved(ctx, &ctx->d_keys[ecdsa], &ctx->d_keys_cap[ecdsa], [&](kgv_carve& c) {
    n_rec = c.take<uint32_t>(64);  // a 256-byte header: the record count
    table = c.take<KeySlot>(slots); item_slot = c.take<uint32_t>(n); rec_rep = c.take<uint32_t>(cap); recs = c.take<uint32_t>(rec_words);
  });
  if (rc) return rc;
  CK(cudaMemsetAsync(n_rec, 0, (uint8_t*)item_slot - (uint8_t*)n_rec, st));  // the header and the slot table
  if (stand_down) {
    k_kc_stand_down<<<1, 1, 0, st>>>(stand_down, n_rec);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  const unsigned gd = (unsigned)((n + 255) / 256);
  // (ECDSA keys, at a 33-byte stride, are never word aligned)
  const auto dedup = ecdsa ? k_key_dedup<false, true> : aligned ? k_key_dedup<true, false> : k_key_dedup<false, false>;
  dedup<<<gd, 256, 0, st>>>(dpk, n, index, n_dev, table, slots - 1, item_slot, rec_rep, n_rec, 0u);
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

// ---- device key cache, host side ----
// A cache is its records, shared by every context attached to it (kgv_keycache_share), and one attachment per context: the streams, events
// and scratch of that context's launches, whose deferred inserts read the scratch of the launch that made them.
//
// Each partition has the UTXO tables' reader/writer lock (kgv_table_sync, ordered on the GPU).  A verify launch READS from its k_kc_lookup to
// the end of its stored-record launch (the stamps and counters it updates are atomics that concurrent readers share); k_kc_insert, at the
// end of a small launch or before a large one verifies (which then holds the write throughout), k_kc_restamp, kgv_keycache_clear and kgv_keycache_counter WRITE.
// So while an insert runs, no launch of any context reads the partition but the inserting launch itself, whose hits carry its stamp: the
// insert's rule (a slot stamped by an earlier launch) keeps what that launch reads, and takes nothing another context still reads.
// Lock order: the partition is taken inside kgv_launch_verify, after any UTXO table the call holds, and no other lock is taken while it is
// held; the Schnorr and ECDSA partitions are never held together.  A registration covers one launch's enqueue, never a whole call, so the
// host synchronisations of a replay window never make another context's insert wait on the host.
struct kgv_keycache_shared {
  struct Part {
    KcPart v{};
    kgv_table_sync sync;                // the partition's lock; its mutex also guards stamp
    uint32_t stamp = 0;                 // stamps handed out so far (the stamp of the last launch)
  } part[2];
  ~kgv_keycache_shared() {              // the last attached context detaches: every launch and insert on it has finished
    for (auto& P : part)
      for (void* p : {(void*)P.v.sets, (void*)P.v.recs, (void*)P.v.ctr}) if (p) cudaFree(p);
  }
};
struct kgv_keycache {
  std::shared_ptr<kgv_keycache_shared> shared;  // its reference count: the attached contexts
  bool enabled = true;                  // kgv_set_keycache, for this context's launches
  struct Part {
    cudaStream_t side = nullptr;        // the second verify launch, and the deferred inserts of small launches
    cudaEvent_t ev_looked_up = nullptr, ev_verified = nullptr, ev_inserted = nullptr;
    cudaEvent_t ev_done = nullptr;      // the end of the last launch of the kind on its caller's stream
    bool pending = false;               // an insert on side that the next launch of the kind waits for
    uint8_t* scratch = nullptr;         // per-launch words, item records, order, miss keys, dedup table
    size_t scratch_cap = 0;
  } part[2];
};

// waits for every launch and insert of this context's attachment (events, not streams: a caller's stream may be gone by then)
static void keycache_quiesce(kgv_keycache* kc) {
  for (auto& P : kc->part) {
    if (P.ev_done) cudaEventSynchronize(P.ev_done);
    if (P.side) cudaStreamSynchronize(P.side);
  }
}
// detaches the context; the records go with the last attached context
static void keycache_free(kgv_ctx* ctx) {
  kgv_keycache* kc = ctx->keycache;
  if (!kc) return;
  keycache_quiesce(kc);
  ctx->keycache = nullptr;
  for (auto& P : kc->part) {
    if (P.scratch) cudaFree(P.scratch);
    for (cudaEvent_t e : {P.ev_looked_up, P.ev_verified, P.ev_inserted, P.ev_done}) if (e) cudaEventDestroy(e);
    if (P.side) cudaStreamDestroy(P.side);
  }
  delete kc;
}
static int keycache_attach(kgv_ctx* ctx, std::shared_ptr<kgv_keycache_shared> shared) {
  ctx->keycache = new kgv_keycache();
  ctx->keycache->shared = std::move(shared);
  for (auto& P : ctx->keycache->part) {
    CK(cudaStreamCreateWithFlags(&P.side, cudaStreamNonBlocking));
    for (cudaEvent_t* e : {&P.ev_looked_up, &P.ev_verified, &P.ev_inserted, &P.ev_done}) CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  }
  return KGV_OK;
}

// Takes partition P's lock for work on st, a write when `write`.  A verify launch gets its stamp here; at the stamps' wrap every used slot
// restarts at 1 (k_kc_restamp), which only a write may do, so a read that meets the wrap is taken again as a write.  A deferred insert
// (insert) stamps with the last stamp handed out, its own launch's when one context uses the cache: no launch reads during an insert, so
// the stamp only keeps the slots of the last launch, of any context, as the most recently used.
static int kc_lock(kgv_ctx* ctx, kgv_table_access& acc, kgv_keycache_shared::Part& P, bool write, cudaStream_t st, bool insert, uint32_t* stamp) {
  for (;;) {
    if (int rc = acc.acquire(&P.sync, write, st)) return rc;
    bool wrap;
    {
      std::lock_guard<std::mutex> g(P.sync.m);
      wrap = !insert && P.stamp + 1 == 0xFFFFFFFFu;
      if (write || !wrap) *stamp = insert ? P.stamp : wrap ? (P.stamp = 2) : ++P.stamp;
    }
    if (!wrap) return KGV_OK;
    if (write) {
      k_kc_restamp<<<nblk(P.v.n_sets, 256), 256, 0, st>>>(P.v.sets, P.v.n_sets);
      CK(cudaGetLastError());
      ctx->launches++;
      return KGV_OK;
    }
    acc.release();
    write = true;
  }
}

struct KcScratch {
  uint32_t *hdr, *item_rec, *order, *miss_order, *item_slot, *rec_rep;
  uint8_t* miss_keys;
  KeySlot* table;
  uint32_t slots;
};
// Starts a launch of the attachment's partition P on st: after the kind's previous insert of this context, with cleared launch words.
// The scratch is sized from the host's n (an upper bound of *n_dev when given) and, like the per-launch key cache's, belongs to the kind.
static int kc_begin(kgv_ctx* ctx, kgv_keycache::Part& P, size_t n, bool ecdsa, cudaStream_t st, KcScratch* s) {
  if (P.pending) CK(cudaStreamWaitEvent(st, P.ev_inserted, 0));
  P.pending = false;
  uint32_t slots = 64;
  while (slots < 2 * n) slots <<= 1;
  int rc = kgv_reserve_carved(ctx, &P.scratch, &P.scratch_cap, [&](kgv_carve& c) {
    s->hdr = c.take<uint32_t>(64);  // the 256-byte header of launch words
    s->item_rec = c.take<uint32_t>(n); s->order = c.take<uint32_t>(n); s->miss_order = c.take<uint32_t>(n); s->miss_keys = c.take<uint8_t>((ecdsa ? 33 : 32) * n);
    s->table = c.take<KeySlot>(slots); s->item_slot = c.take<uint32_t>(n); s->rec_rep = c.take<uint32_t>(n);
  });
  if (rc) return rc;
  s->slots = slots;
  CK(cudaMemsetAsync(s->hdr, 0, 256, st));
  return KGV_OK;
}
// the insert of a launch's misses into partition p on st: k_key_dedup over the miss keys, then k_kc_insert
static int kc_insert(kgv_ctx* ctx, const KcPart& p, const KcScratch& s, size_t n, bool ecdsa, cudaStream_t st, uint32_t stamp, bool gate) {
  CK(cudaMemsetAsync(s.table, 0, (size_t)s.slots * sizeof(KeySlot), st));
  // (the miss keys are packed from a 256-byte aligned base: Schnorr's are word aligned)
  // a large launch's insert takes at most the partition's slots and KGV_KEY_RECORDS_MAX keys (k_kc_insert's gate): past that many the
  // dedup stops, the gate refuses the launch
  const uint32_t slots = p.n_sets * KGV_KC_WAYS, limit = gate ? std::min(slots, (uint32_t)KGV_KEY_RECORDS_MAX) : 0xFFFFFFFFu;
  const auto dedup = ecdsa ? k_key_dedup<false, true, true> : k_key_dedup<true, false, true>;
  dedup<<<nblk(n, 256), 256, 0, st>>>(s.miss_keys, n, nullptr, s.hdr + KC_N_MISS, s.table, s.slots - 1, s.item_slot, s.rec_rep, s.hdr + KC_N_REC,
                                      limit);
  CK(cudaGetLastError());
  const auto insert = ecdsa ? k_kc_insert<true> : k_kc_insert<false>;
  insert<<<nblk(n, KGV_BLOCK), KGV_BLOCK, 0, st>>>(p, s.miss_keys, s.rec_rep, s.hdr, stamp, gate);
  CK(cudaGetLastError());
  ctx->launches += 2;
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
  // With a device key cache (kgv_keycache) the items whose keys are stored are verified from their comb records by one launch on st, the
  // others by a second launch, of the form they take without the cache, on the partition's side stream at the same time; st waits for
  // it.  A small launch stores its misses afterwards on the side stream, off the call's path; a large one stores them first when its insert
  // takes the launch (k_kc_insert), else every item goes to the second launch, which then runs as without the cache.
  kgv_keycache* cache = ctx->keycache;
  kgv_keycache_shared::Part* sp = cache && cache->enabled && cache->shared->part[ecdsa].v.n_sets ? &cache->shared->part[ecdsa] : nullptr;
  if (!index) {
    auto& lv = ctx->last_verify[ecdsa];
    lv.n = n; lv.blocks = blocks; lv.key_cache = key_cache && !sp; lv.stream = st;
  }
  if (!sp) {
    if (key_cache) {
      int rc = key_cache_launch(ctx, dpk, n, ecdsa, aligned, st, index, n_dev, &kc);
      if (rc) return rc;
    }
    k_verify[ecdsa][index != nullptr][aligned]<<<blocks, KGV_BLOCK, smem, st>>>(dpk, dmsg, dsig, n, dst, ctx->gtab, index, n_dev, kc);
    CK(cudaGetLastError());
    ctx->launches++;
    return KGV_OK;
  }
  kgv_keycache::Part* kp = &cache->part[ecdsa];
  KcScratch ks{};
  if (int rc = kc_begin(ctx, *kp, n, ecdsa, st, &ks)) return rc;
  kgv_table_access acc(ctx);
  uint32_t stamp;
  if (int rc = kc_lock(ctx, acc, *sp, key_cache, st, false, &stamp)) return rc;
  const auto lookup = ecdsa ? k_kc_lookup<false, true> : aligned ? k_kc_lookup<true, false> : k_kc_lookup<false, false>;
  lookup<<<nblk(n, 256), 256, 0, st>>>(dpk, n, index, n_dev, sp->v, stamp, key_cache ? KC_COUNT : KC_COUNT | KC_ORDER, ks.hdr, ks.item_rec,
                                       ks.order, ks.miss_order, ks.miss_keys);
  CK(cudaGetLastError());
  ctx->launches++;
  if (key_cache) {
    if (int rc = kc_insert(ctx, sp->v, ks, n, ecdsa, st, stamp, true)) return rc;
    if (int rc = key_cache_launch(ctx, dpk, n, ecdsa, aligned, st, index, n_dev, &kc, ks.hdr)) return rc;
    lookup<<<nblk(n, 256), 256, 0, st>>>(dpk, n, index, n_dev, sp->v, stamp, KC_ORDER | KC_GATED, ks.hdr, ks.item_rec, ks.order, ks.miss_order,
                                         ks.miss_keys);
    CK(cudaGetLastError());
    ctx->launches++;
  }
  CK(cudaEventRecord(kp->ev_looked_up, st));
  CK(cudaStreamWaitEvent(kp->side, kp->ev_looked_up, 0));
  KeyCacheView stored{};
  stored.item_rec = ks.item_rec;
  stored.kc_recs = sp->v.recs;
  k_verify[ecdsa][1][aligned]<<<blocks, KGV_BLOCK, smem, st>>>(dpk, dmsg, dsig, n, dst, ctx->gtab, ks.order, ks.hdr + KC_ORD_HIT, stored);
  CK(cudaGetLastError());
  acc.release();  // the last read of the partition's records
  k_verify[ecdsa][1][aligned]<<<blocks, KGV_BLOCK, smem, kp->side>>>(dpk, dmsg, dsig, n, dst, ctx->gtab, ks.miss_order, ks.hdr + KC_ORD_MISS, kc);
  CK(cudaGetLastError());
  ctx->launches += 2;
  CK(cudaEventRecord(kp->ev_verified, kp->side));
  CK(cudaStreamWaitEvent(st, kp->ev_verified, 0));
  CK(cudaEventRecord(kp->ev_done, st));
  if (!key_cache) {
    if (int rc = kc_lock(ctx, acc, *sp, true, kp->side, true, &stamp)) return rc;
    if (int rc = kc_insert(ctx, sp->v, ks, n, ecdsa, kp->side, stamp, false)) return rc;
    acc.release();
    CK(cudaEventRecord(kp->ev_inserted, kp->side));
    kp->pending = true;
  }
  return KGV_OK;
}

extern "C" int kgv_keycache_create(kgv_ctx* ctx, uint64_t schnorr_keys, uint64_t ecdsa_keys) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (ctx->keycache) return fail_arg(ctx, "kgv_keycache_create: the context has a key cache");
  if (schnorr_keys == 0 && ecdsa_keys == 0) return fail_arg(ctx, "kgv_keycache_create: both capacities are 0");
  if (schnorr_keys > KGV_KEYCACHE_MAX_KEYS || ecdsa_keys > KGV_KEYCACHE_MAX_KEYS)
    return fail_arg(ctx, "kgv_keycache_create: a capacity above KGV_KEYCACHE_MAX_KEYS");
  CK(cudaSetDevice(ctx->device));
  auto shared = std::make_shared<kgv_keycache_shared>();
  for (int k = 0; k < 2; k++) {
    auto& P = shared->part[k];
    P.sync.device = ctx->device;
    const uint64_t keys = k ? ecdsa_keys : schnorr_keys;
    if (!keys) continue;
    const uint32_t n_sets = (uint32_t)((keys + KGV_KC_WAYS - 1) / KGV_KC_WAYS);
    if (int rc = kgv_malloc(ctx, (void**)&P.v.sets, (size_t)n_sets * sizeof(KcSet))) return rc;
    if (int rc = kgv_malloc(ctx, (void**)&P.v.recs, (size_t)n_sets * KGV_KC_WAYS * KGV_JR_WORDS * 4)) return rc;
    if (int rc = kgv_malloc(ctx, (void**)&P.v.ctr, 4 * sizeof(unsigned long long))) return rc;
    P.v.n_sets = n_sets;
    CK(cudaMemsetAsync(P.v.sets, 0, (size_t)n_sets * sizeof(KcSet), ctx->stream));
    CK(cudaMemsetAsync(P.v.ctr, 0, 4 * sizeof(unsigned long long), ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  if (int rc = keycache_attach(ctx, std::move(shared))) {
    keycache_free(ctx);
    return rc;
  }
  return KGV_OK;
}

extern "C" int kgv_keycache_share(kgv_ctx* ctx, kgv_ctx* holder) {
  if (!ctx || !holder) return KGV_ERR_ARG;
  if (ctx == holder) return fail_arg(ctx, "kgv_keycache_share: ctx and holder are the same context");
  std::scoped_lock g(ctx->mu, holder->mu);
  if (!holder->keycache) return fail_arg(ctx, "kgv_keycache_share: the holder has no key cache");
  if (ctx->keycache) return fail_arg(ctx, "kgv_keycache_share: the context has a key cache");
  if (ctx->device != holder->device) {
    ctx->err = "kgv_keycache_share: the holder's cache is on device " + std::to_string(holder->device) + ", the context on device " +
               std::to_string(ctx->device);
    return KGV_ERR_ARG;
  }
  CK(cudaSetDevice(ctx->device));
  if (int rc = keycache_attach(ctx, holder->keycache->shared)) {
    keycache_free(ctx);
    return rc;
  }
  return KGV_OK;
}

extern "C" int kgv_keycache_destroy(kgv_ctx* ctx) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  keycache_free(ctx);
  return KGV_OK;
}

// a write on each partition in turn: it waits for the launches and inserts of every attached context enqueued before it
extern "C" int kgv_keycache_clear(kgv_ctx* ctx) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  kgv_keycache* kc = ctx->keycache;
  if (!kc) return fail_arg(ctx, "kgv_keycache_clear: the context has no key cache");
  CK(cudaSetDevice(ctx->device));
  for (auto& P : kc->shared->part) {
    if (!P.v.n_sets) continue;
    kgv_table_access acc(ctx);
    if (int rc = acc.acquire(&P.sync, true, ctx->stream)) return rc;
    CK(cudaMemsetAsync(P.v.sets, 0, (size_t)P.v.n_sets * sizeof(KcSet), ctx->stream));
    CK(cudaMemsetAsync(P.v.ctr, 0, 4 * sizeof(unsigned long long), ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  return KGV_OK;
}

// read under a write, so that the value covers the launches of every attached context enqueued before the call
extern "C" uint64_t kgv_keycache_counter(kgv_ctx* ctx, int ecdsa, int which) {
  if (!ctx) return 0;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  kgv_keycache* kc = ctx->keycache;
  if (!kc || which < 0 || which > 3) return 0;
  const int k = ecdsa ? 1 : 0;
  auto& P = kc->shared->part[k];
  if (!P.v.n_sets) return 0;
  unsigned long long v = 0;
  const cudaStream_t side = kc->part[k].side;
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e == cudaSuccess) {
    kgv_table_access acc(ctx);
    if (acc.acquire(&P.sync, true, side)) return UINT64_MAX;
    e = cudaMemcpyAsync(&v, P.v.ctr + which, sizeof v, cudaMemcpyDeviceToHost, side);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(side);
  if (e != cudaSuccess) {
    ctx->err = std::string("kgv_keycache_counter: ") + cudaGetErrorString(e);
    (void)cudaGetLastError();
    return UINT64_MAX;
  }
  return v;
}

extern "C" int kgv_set_keycache(kgv_ctx* ctx, int enabled) {
  if (!ctx) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (!ctx->keycache) return fail_arg(ctx, "kgv_set_keycache: the context has no key cache");
  ctx->keycache->enabled = enabled != 0;
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
    uint8_t *dpk, *dmsg;
    // the messages, and the signatures straight after them
    int rc = kgv_reserve_carved(ctx, &ctx->d_in, &ctx->d_in_cap, [&](kgv_carve& c) { dpk = c.take<uint8_t>(pk_stride * n); dmsg = c.take<uint8_t>(96 * n); });
    if (rc) return rc;
    uint8_t* dsig = dmsg + 32 * n;
    rc = kgv_reserve(ctx, &ctx->d_out, &ctx->d_out_cap, n);
    if (rc) return rc;
    uint8_t* dst = ctx->d_out;
    CK(cudaEventRecord(ctx->ev_fork, ctx->stream));          // the staging buffers may still be read by earlier work of this stream
    CK(cudaStreamWaitEvent(ctx->aux_stream, ctx->ev_fork, 0));
    size_t c = 0;
    for (size_t a = 0; a < n; a += chunk, c++) {
      const size_t m = n - a < chunk ? n - a : chunk;
      if (!ctx->ev_chunk[c]) CK(cudaEventCreateWithFlags(&ctx->ev_chunk[c], cudaEventDisableTiming));
      CK(cudaMemcpyAsync(dpk + pk_stride * a, pk + pk_stride * a, pk_stride * m, cudaMemcpyHostToDevice, ctx->aux_stream));
      CK(cudaMemcpyAsync(dmsg + 32 * a, msg + 32 * a, 32 * m, cudaMemcpyHostToDevice, ctx->aux_stream));
      CK(cudaMemcpyAsync(dsig + 64 * a, sig + 64 * a, 64 * m, cudaMemcpyHostToDevice, ctx->aux_stream));
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
