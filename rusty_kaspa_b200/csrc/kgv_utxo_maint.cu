// kgv_utxo_maint.cu — maintenance of the GPU UTXO table (K5, kgv_utxo.cuh): stats, out-of-place rehash and the opt-in growth policy.
//
// The probing scheme is untouched: linear probing, erase = tombstone, an insert reuses the first tombstone before the first EMPTY slot.  Under
// churn EMPTY slots turn into tombstones and never come back, so misses and inserts probe ever longer runs; the rehash moves every entry
// into a fresh array (tombstones dropped, long scripts compacted) and the policy does that before a write would overfill the table.
#include "kgv_internal.h"
#include "kgv_utxo.cuh"

#include <cstdio>

using namespace kgv;


// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
// A range of consecutive slots as the longest-run reduction sees it: its length, the non-EMPTY runs touching its two edges and the longest
// run inside.  The range is all occupied when pre == len.  Joining is associative, so blocks reduce in order and a last step adds the
// wrap-around (the suffix run of the table continues into its prefix run).
struct RunSeg {
  unsigned long long len, pre, suf, best;
};
__device__ __forceinline__ RunSeg run_join(const RunSeg& a, const RunSeg& b) {  // a lies left of b
  RunSeg r;
  r.len = a.len + b.len;
  r.pre = a.pre == a.len ? a.len + b.pre : a.pre;
  r.suf = b.suf == b.len ? b.len + a.suf : b.suf;
  r.best = max(max(a.best, b.best), a.suf + b.pre);
  return r;
}
__device__ __forceinline__ RunSeg run_shfl_down(const RunSeg& s, int o) {
  RunSeg r;
  r.len = __shfl_down_sync(0xFFFFFFFFu, s.len, o);
  r.pre = __shfl_down_sync(0xFFFFFFFFu, s.pre, o);
  r.suf = __shfl_down_sync(0xFFFFFFFFu, s.suf, o);
  r.best = __shfl_down_sync(0xFFFFFFFFu, s.best, o);
  return r;
}
// ordered join of one segment per thread (thread order = slot order); the result is valid in thread 0.  w_seg: one RunSeg per warp.
__device__ __forceinline__ RunSeg block_run_join(RunSeg s, RunSeg* w_seg) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const RunSeg r = run_shfl_down(s, o);
    if ((lane & (2 * o - 1)) == 0) s = run_join(s, r);
  }
  if (lane == 0) w_seg[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) s = run_join(s, w_seg[w]);
  return s;
}
__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
  return v;
}
__device__ __forceinline__ unsigned long long warp_max(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_down_sync(0xFFFFFFFFu, v, o));
  return v;
}

#define STATS_THREADS 256
#define STATS_ITEMS 4  // consecutive slots per thread: STATS_THREADS * STATS_ITEMS = 1024 slots per block, the smallest table
enum { ACC_EMPTY, ACC_LIVE, ACC_LONG_BYTES, ACC_SUM_DISP, ACC_MAX_DISP, ACC_LONGEST_RUN, ACC_WORDS = 8 };

// One pass over the slot heads (64 bytes each, slot_load_head): EMPTY slots, entries (FULL / FULLH / REMOVED), their displacement from the
// home slot and the padded bytes of their long scripts into acc[]; the block's run segment into segs[blockIdx.x].
__global__ void __launch_bounds__(STATS_THREADS) k_utxo_stats(TableView t, unsigned long long* __restrict__ acc, RunSeg* __restrict__ segs) {
  __shared__ RunSeg w_seg[STATS_THREADS / 32];
  __shared__ unsigned long long s_acc[ACC_LONGEST_RUN];
  if (threadIdx.x < ACC_LONGEST_RUN) s_acc[threadIdx.x] = 0;
  const uint64_t first = ((uint64_t)blockIdx.x * STATS_THREADS + threadIdx.x) * STATS_ITEMS;
  unsigned long long n_empty = 0, n_live = 0, long_bytes = 0, sum_d = 0, max_d = 0, cur = 0;
  RunSeg seg{STATS_ITEMS, 0, 0, 0};
  bool seen_empty = false;
#pragma unroll
  for (int j = 0; j < STATS_ITEMS; j++) {
    const uint64_t i = first + j;
    SlotHead h;
    slot_load_head(h, &t.slots[i]);
    const uint32_t st = h.state();
    if (st == SLOT_EMPTY) {
      n_empty++;
      if (!seen_empty) seg.pre = cur;
      seen_empty = true;
      seg.best = max(seg.best, cur);
      cur = 0;
      continue;
    }
    cur++;
    if (st == SLOT_FULL || st >= SLOT_REMOVED) {
      n_live++;
      const unsigned long long d = (i - key_hash(h.w + 1)) & t.mask;
      sum_d += d;
      max_d = max(max_d, d);
      const uint32_t len = h.meta() >> 17;
      if (len > INLINE_SCRIPT) long_bytes += (len + 7u) & ~7u;
    }
  }
  if (!seen_empty) seg.pre = seg.suf = seg.best = STATS_ITEMS;
  else { seg.suf = cur; seg.best = max(seg.best, cur); }
  n_empty = warp_sum(n_empty); n_live = warp_sum(n_live); long_bytes = warp_sum(long_bytes); sum_d = warp_sum(sum_d); max_d = warp_max(max_d);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&s_acc[ACC_EMPTY], n_empty); atomicAdd(&s_acc[ACC_LIVE], n_live); atomicAdd(&s_acc[ACC_LONG_BYTES], long_bytes);
    atomicAdd(&s_acc[ACC_SUM_DISP], sum_d); atomicMax(&s_acc[ACC_MAX_DISP], max_d);
  }
  seg = block_run_join(seg, w_seg);  // (its barrier also orders the shared accumulators)
  if (threadIdx.x == 0) {
    segs[blockIdx.x] = seg;
    atomicAdd(&acc[ACC_EMPTY], s_acc[ACC_EMPTY]); atomicAdd(&acc[ACC_LIVE], s_acc[ACC_LIVE]); atomicAdd(&acc[ACC_LONG_BYTES], s_acc[ACC_LONG_BYTES]);
    atomicAdd(&acc[ACC_SUM_DISP], s_acc[ACC_SUM_DISP]); atomicMax(&acc[ACC_MAX_DISP], s_acc[ACC_MAX_DISP]);
  }
}
// second step, one block: the blocks' segments joined in order, then the wrap-around
__global__ void __launch_bounds__(1024) k_utxo_stats_join(const RunSeg* __restrict__ segs, uint32_t n, unsigned long long* __restrict__ acc) {
  __shared__ RunSeg w_seg[32];
  const uint32_t per = (n + blockDim.x - 1) / blockDim.x, lo = min(n, threadIdx.x * per), hi = min(n, lo + per);
  RunSeg s{0, 0, 0, 0};
  for (uint32_t b = lo; b < hi; b++) s = run_join(s, segs[b]);
  s = block_run_join(s, w_seg);
  if (threadIdx.x == 0) acc[ACC_LONGEST_RUN] = s.pre == s.len ? s.len : max(s.best, s.suf + s.pre);
}

// One thread per old slot.  Entries (FULL, FULLH, REMOVED) move with their state; TOMB and EMPTY are dropped.  The keys are distinct, so an
// entry takes the first EMPTY slot from its home slot (atomicCAS on the state word) with no key compare and no tombstone logic.  A long
// script is bump-allocated in the new arena (counters[2], zeroed by the host) and its offset word rewritten.  The new array is sized so
// that every entry and every script fits; a failure would still be counted in counters[3].
__global__ void __launch_bounds__(256) k_utxo_rehash(TableView old, UtxoSlot* __restrict__ slots, uint64_t mask, uint8_t* __restrict__ overflow,
                                                     uint64_t overflow_cap, unsigned long long* __restrict__ counters) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > old.mask) return;
  const UtxoSlot* s = &old.slots[i];
  uint32_t w[32];
  ld256_cg(w, s);
  const uint32_t st = w[0];
  if (st != SLOT_FULL && st < SLOT_REMOVED) return;
  ld256_cg(w + 8, (const uint8_t*)s + 32);
  ld256_cg(w + 16, (const uint8_t*)s + 64);
  ld256_cg(w + 24, (const uint8_t*)s + 96);
  const uint32_t len = w[14] >> 17;
  if (len > INLINE_SCRIPT) {
    const uint64_t need = (len + 7u) & ~7ull;
    const uint64_t off = atomicAdd(&counters[2], (unsigned long long)need);
    if (off + need > overflow_cap) { atomicAdd(&counters[3], 1ull); return; }
    const uint64_t* src = (const uint64_t*)(old.overflow + ((uint64_t)w[16] << 32 | w[15]));  // offsets and sizes are multiples of 8
    uint64_t* dst = (uint64_t*)(overflow + off);
    for (uint64_t q = 0; q < need / 8; q++) dst[q] = __ldcg(src + q);
    w[15] = (uint32_t)off; w[16] = (uint32_t)(off >> 32);
  }
  uint64_t j = key_hash(w + 1) & mask;
  for (uint64_t probes = 0;; probes++, j = (j + 1) & mask) {
    if (probes > mask) { atomicAdd(&counters[3], 1ull); return; }
    if (atomicCAS(&slots[j].state, SLOT_EMPTY, st) == SLOT_EMPTY) break;
  }
  UtxoSlot* d = &slots[j];
  st256(d, w);
  st256((uint8_t*)d + 32, w + 8);
  st256((uint8_t*)d + 64, w + 16);
  st256((uint8_t*)d + 96, w + 24);
}

// ---------------------------------------------------------------------------------------------
// host side: the calls of several contexts on one table (kgv_internal.h)
// ---------------------------------------------------------------------------------------------
static int pooled_event(kgv_table_sync* s, cudaEvent_t* ev) {  // (s->m held)
  if (!s->pool.empty()) { *ev = s->pool.back(); s->pool.pop_back(); return KGV_OK; }
  return cudaEventCreateWithFlags(ev, cudaEventDisableTiming) == cudaSuccess ? KGV_OK : KGV_ERR_CUDA;
}

kgv_table_sync::~kgv_table_sync() {
  for (const auto& r : reads) cudaEventDestroy(r.second);
  for (const auto& r : retired) cudaEventDestroy(r.done);
  for (cudaEvent_t e : pool) cudaEventDestroy(e);
  for (cudaEvent_t e : {last_write, retire_ev}) if (e) cudaEventDestroy(e);
}

int kgv_table_access::lock(kgv_table_sync* s, Mode m, cudaStream_t st) {
  std::unique_lock<std::mutex> g(s->m);
  Held h{s, m, nullptr, st};
  if (s->writer == ctx && s->write_depth > 0) {  // nested in this context's own write
    if (m == kWrite) s->write_depth++;
    else h.m = kNone;
    held.push_back(h);
    return KGV_OK;
  }
  cudaError_t e = cudaSuccess;
  if (m == kRead) {
    auto it = s->readers.begin();
    while (it != s->readers.end() && it->ctx != ctx) ++it;
    if (it != s->readers.end()) {  // nested in a read of this context: a queued writer waits for it, so this must not wait for the writer
      it->depth++;
      held.push_back(h);
      return KGV_OK;
    }
    if (pooled_event(s, &h.ev)) { ctx->err = "cudaEventCreate failed for a table read"; return KGV_ERR_CUDA; }
    s->cv.wait(g, [&] { return s->write_depth == 0 && s->next_ticket == s->serving; });
    s->readers.push_back({ctx, 1});
    if (s->last_write) e = cudaStreamWaitEvent(st, s->last_write, 0);
  } else {
    if (!s->last_write && pooled_event(s, &s->last_write)) { ctx->err = "cudaEventCreate failed for a table write"; return KGV_ERR_CUDA; }
    const uint64_t ticket = s->next_ticket++;
    s->cv.wait(g, [&] {
      if (s->serving != ticket || s->write_depth) return false;
      for (const auto& r : s->readers) if (r.ctx != ctx) return false;
      return true;
    });
    s->writer = ctx;
    s->write_depth = 1;
    for (const auto& r : s->reads) {
      if (e == cudaSuccess) e = cudaStreamWaitEvent(st, r.second, 0);
      s->pool.push_back(r.second);
    }
    s->reads.clear();
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, s->last_write, 0);
  }
  held.push_back(h);  // held from here on, so that release() undoes it even when the wait failed
  if (e != cudaSuccess) { ctx->err = std::string("ordering a table access: ") + cudaGetErrorString(e); return KGV_ERR_CUDA; }
  return KGV_OK;
}

int kgv_table_access::acquire(const char* call, kgv_utxo_table* t, kgv_utxo_table* written) {
  kgv_utxo_table* chain[64];
  int n = 0;
  for (kgv_utxo_table* L = t; L; L = L->base) {
    if (n == 64) { ctx->err = std::string(call) + ": a view chain deeper than 64 layers"; return KGV_ERR_LIMIT; }
    if (L->sync->device != ctx->device) {
      ctx->err = std::string(call) + ": the UTXO table belongs to device " + std::to_string(L->sync->device) + ", the context to device " +
                 std::to_string(ctx->device);
      return KGV_ERR_ARG;
    }
    chain[n++] = L;
  }
  while (n--)
    if (int rc = lock(chain[n]->sync.get(), chain[n] == written ? kWrite : kRead, ctx->stream)) return rc;
  return KGV_OK;
}

int kgv_table_access::acquire(kgv_table_sync* s, bool write, cudaStream_t st) { return lock(s, write ? kWrite : kRead, st); }

void kgv_table_access::release() {
  while (!held.empty()) {
    Held h = held.back();
    held.pop_back();
    kgv_table_sync* s = h.s;
    const cudaStream_t st = h.st;
    std::lock_guard<std::mutex> g(s->m);
    if (h.m == kWrite) {
      if (--s->write_depth) continue;
      cudaEventRecord(s->last_write, st);
      s->writes++;
      if (!s->retiring.empty()) {
        cudaEventRecord(s->retire_ev, st);
        s->retired.push_back({s->retire_ev, std::move(s->retiring)});
        s->retiring.clear();
        s->retire_ev = nullptr;
      }
      s->writer = nullptr;
      s->serving++;
    } else if (h.m == kRead) {
      auto it = s->readers.begin();
      while (it != s->readers.end() && it->ctx != ctx) ++it;
      if (it == s->readers.end() || --it->depth) continue;
      s->readers.erase(it);
      cudaEvent_t ev = h.ev;
      for (auto& r : s->reads)  // a later record on the same stream supersedes the earlier one
        if (r.first == st) { s->pool.push_back(ev); ev = r.second; break; }
      if (ev == h.ev) s->reads.push_back({st, ev});
      cudaEventRecord(ev, st);
    } else {
      continue;
    }
    s->cv.notify_all();
  }
}

int kgv_table_retire(kgv_ctx* ctx, kgv_utxo_table* t, void* p) {
  kgv_table_sync* s = t->sync.get();
  std::lock_guard<std::mutex> g(s->m);
  if (!s->retire_ev && pooled_event(s, &s->retire_ev)) {
    ctx->err = "cudaEventCreate failed for a released table array";
    return KGV_ERR_CUDA;
  }
  s->retiring.push_back(p);
  for (const auto& r : ctx->retiring) if (r.get() == s) return KGV_OK;
  ctx->retiring.push_back(t->sync);
  return KGV_OK;
}

void kgv_release_retired(kgv_ctx* ctx, bool wait) {
  auto& v = ctx->retiring;
  for (size_t i = 0; i < v.size();) {
    kgv_table_sync* s = v[i].get();
    bool empty;
    {
      std::lock_guard<std::mutex> g(s->m);
      auto& R = s->retired;
      for (size_t j = 0; j < R.size();) {
        if (wait) cudaEventSynchronize(R[j].done);
        if (cudaEventQuery(R[j].done) != cudaSuccess) { (void)cudaGetLastError(); j++; continue; }
        for (void* p : R[j].ptrs) cudaFree(p);
        s->pool.push_back(R[j].done);
        R.erase(R.begin() + j);
      }
      empty = R.empty() && s->retiring.empty();
    }
    if (empty) v.erase(v.begin() + i);
    else i++;
  }
}

uint64_t kgv_chain_rehashes(const kgv_utxo_table* t) {
  uint64_t n = 0;
  for (; t; t = t->base) n += t->rehashes;
  return n;
}

int kgv_last_replay_read(kgv_ctx* ctx, kgv_table_access& acc, const char* call) {
  if (int rc = acc.acquire(call, ctx->last_replay.table)) return rc;
  if (kgv_chain_rehashes(ctx->last_replay.table) == ctx->last_replay.rehashes) return KGV_OK;
  ctx->last_replay.valid = false;
  ctx->err = std::string(call) + " refers to the last kgv_replay_window call, and its table was rehashed since";
  return KGV_ERR_ARG;
}

// ---------------------------------------------------------------------------------------------
// host side: maintenance
// ---------------------------------------------------------------------------------------------
// counters + one stats pass; synchronises
static int utxo_scan(kgv_ctx* ctx, kgv_utxo_table* t, kgv_utxo_table_stats* out, uint64_t* n_entries) {
  const uint64_t cap = t->mask + 1;
  const uint32_t n_blocks = (uint32_t)(cap / (STATS_THREADS * STATS_ITEMS));
  const size_t o_segs = ACC_WORDS * sizeof(unsigned long long);
  int rc = kgv_reserve(ctx, &ctx->d_work, &ctx->d_work_cap, o_segs + (size_t)n_blocks * sizeof(RunSeg));
  if (rc) return rc;
  unsigned long long* acc = (unsigned long long*)ctx->d_work;
  RunSeg* segs = (RunSeg*)(ctx->d_work + o_segs);
  cudaStream_t st = ctx->stream;
  CK(cudaMemsetAsync(acc, 0, o_segs, st));
  k_utxo_stats<<<n_blocks, STATS_THREADS, 0, st>>>(view_of(t), acc, segs);
  CK(cudaGetLastError());
  k_utxo_stats_join<<<1, 1024, 0, st>>>(segs, n_blocks, acc);
  CK(cudaGetLastError());
  ctx->launches += 2;
  unsigned long long a[ACC_WORDS], c[4];
  CK(cudaMemcpyAsync(a, acc, sizeof a, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(c, t->counters, sizeof c, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  out->capacity_slots = cap;
  out->live = c[0];
  out->tombstones = c[1];
  out->empty = a[ACC_EMPTY];
  out->overflow_used = c[2];
  out->overflow_cap = t->overflow_cap;
  out->overflow_live = a[ACC_LONG_BYTES];
  out->insert_failures = c[3];
  out->rehashes = t->rehashes;
  out->max_displacement = a[ACC_MAX_DISP];
  out->sum_displacement = a[ACC_SUM_DISP];
  out->longest_run = a[ACC_LONGEST_RUN];
  if (n_entries) *n_entries = a[ACC_LIVE];
  return KGV_OK;
}

static const uint64_t kMaxCapacity = 1ull << 40;

// arena_headroom: long-script bytes the caller is about to append (the growth policy), on top of the live ones
static int utxo_rehash(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t capacity_slots, uint64_t arena_headroom) {
  if (capacity_slots > kMaxCapacity) { ctx->err = "kgv_utxo_rehash: capacity too large"; return KGV_ERR_ARG; }
  kgv_utxo_table_stats s;
  uint64_t n_entries = 0;
  int rc = utxo_scan(ctx, t, &s, &n_entries);
  if (rc) return rc;
  const uint64_t want = capacity_slots ? capacity_slots : t->mask + 1;
  uint64_t cap = 1024;
  while (cap < want) cap <<= 1;
  if (cap < s.live + 1 || cap < n_entries + 1) { ctx->err = "kgv_utxo_rehash: the capacity must exceed the live entries"; return KGV_ERR_ARG; }
  uint64_t arena = cap * 8 < (64ull << 20) ? (64ull << 20) : cap * 8;  // as kgv_utxo_create, and room for the live scripts twice over
  if (arena < 2 * s.overflow_live) arena = 2 * s.overflow_live;
  if (arena < s.overflow_live + arena_headroom) arena = s.overflow_live + arena_headroom;
  UtxoSlot* slots = nullptr;
  uint8_t* overflow = nullptr;
  rc = kgv_malloc(ctx, (void**)&slots, cap * sizeof(UtxoSlot));
  if (rc) return rc;
  rc = kgv_malloc(ctx, (void**)&overflow, arena);
  if (rc) { ctx->parked.push_back((uint8_t*)slots); return rc; }  // (no cudaFree inside a call: see kgv_reserve)
  cudaStream_t st = ctx->stream;
  CK(cudaMemsetAsync(slots, 0, cap * sizeof(UtxoSlot), st));
  CK(cudaMemsetAsync(t->counters + 1, 0, 2 * sizeof(unsigned long long), st));  // tombstones, arena bytes: rebuilt by the kernel
  k_utxo_rehash<<<nblk(t->mask + 1, 256), 256, 0, st>>>(view_of(t), slots, cap - 1, overflow, arena, t->counters);
  CK(cudaGetLastError());
  ctx->launches++;
  // the old arrays may still be read by work queued before this write, of any context: released once the write has completed
  if ((rc = kgv_table_retire(ctx, t, t->slots)) || (rc = kgv_table_retire(ctx, t, t->overflow))) return rc;
  t->slots = slots;
  t->mask = cap - 1;
  t->overflow = overflow;
  t->overflow_cap = arena;
  const TableView hv = view_of(t);  // what view layers above reach through `below`, rewritten in stream order
  CK(cudaMemcpyAsync(t->d_view, &hv, sizeof hv, cudaMemcpyHostToDevice, st));
  t->rehashes++;
  t->occ_bound = s.live;
  t->arena_bound = s.overflow_live;
  // the entries kgv_replay_window staged for kgv_replay_muhash point into the old arena
  ctx->last_replay.valid = false;
  return KGV_OK;
}

int utxo_reserve(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t m, uint64_t b) {
  if (!t->max_load) return KGV_OK;
  const uint64_t cap = t->mask + 1, limit = cap * t->max_load / 1000;
  if (t->occ_bound + m <= limit && t->arena_bound + b <= t->overflow_cap) {
    t->occ_bound += m;
    t->arena_bound += b;
    return KGV_OK;
  }
  unsigned long long c[3];
  CK(cudaMemcpyAsync(c, t->counters, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  const uint64_t live = c[0], occupied = c[0] + c[1], used = c[2];
  uint64_t new_cap = 0;
  if (live + m > limit) {
    new_cap = cap;
    while ((live + m) * 2000 > new_cap * t->max_load) new_cap <<= 1;
  } else if (occupied + m > limit || used + b > t->overflow_cap) {
    new_cap = cap;
  }
  if (!new_cap) {
    t->occ_bound = occupied + m;
    t->arena_bound = used + b;
    return KGV_OK;
  }
  int rc = utxo_rehash(ctx, t, new_cap, b);
  if (rc) return rc;
  t->occ_bound += m;
  t->arena_bound += b;
  return KGV_OK;
}

extern "C" int kgv_utxo_stats(kgv_ctx* ctx, kgv_utxo_table* t, kgv_utxo_table_stats* out) {
  if (!ctx || !t || !out) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (int rc = kgv_host_only(ctx, "kgv_utxo_stats", "out", out)) return rc;
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_stats", t)) return rc;
  return utxo_scan(ctx, t, out, nullptr);
}

extern "C" int kgv_utxo_rehash(kgv_ctx* ctx, kgv_utxo_table* t, uint64_t capacity_slots) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_rehash", t, t)) return rc;
  return utxo_rehash(ctx, t, capacity_slots, 0);
}

extern "C" int kgv_utxo_set_max_load(kgv_ctx* ctx, kgv_utxo_table* t, uint32_t max_load_permille) {
  if (!ctx || !t) return KGV_ERR_ARG;
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  if (max_load_permille > 900) { ctx->err = "max_load_permille: 0 (off) or 1..900"; return KGV_ERR_ARG; }
  CK(cudaSetDevice(ctx->device));
  kgv_table_access acc(ctx);
  if (int rc = acc.acquire("kgv_utxo_set_max_load", t, t)) return rc;
  t->max_load = max_load_permille;
  if (max_load_permille) {  // start the host-side bounds from the exact values
    unsigned long long c[3];
    CK(cudaMemcpyAsync(c, t->counters, sizeof c, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    t->occ_bound = c[0] + c[1];
    t->arena_bound = c[2];
  }
  return KGV_OK;
}
