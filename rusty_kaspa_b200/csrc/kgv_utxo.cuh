// kgv_utxo.cuh — device side of the GPU-resident UTXO set (K5): open addressing, linear probing, one 128-byte slot per
// entry = one L2 line = four 32-byte DRAM sectors.  Plays the role of DbUtxoSetStore / UtxoCollection behind UtxoView::get
// (consensus/src/model/stores/utxo_set.rs:143-152, consensus/core/src/utxo/utxo_collection.rs:28-32).
//
// Memory traffic is the whole cost of this stage, so every slot access is a 128-bit vector access:
//   key      36 bytes at a 4-byte aligned address: nine 32-bit loads (a warp's keys are 1 152 contiguous bytes)
//   probe    the first 64 bytes of a slot (state, outpoint, amount, DAA score, meta, 4 script bytes) with four LDG.128
//            issued back to back: ONE memory round trip per probe, and everything the UTXO-context rules need;
//            the remaining 64 script bytes are read by whoever hashes / parses the script (pointer into the slot)
//   insert   eight STG.128 + one release store of the state word
// Slot loads are L2-coherent (ld.global.cg: the table is written by other SMs of the same launch), never L1 cached
// (random 128-byte accesses have no L1 reuse).
#pragma once
#include <memory>

#include "kgv_script_std.cuh"

#define SLOT_EMPTY 0u
#define SLOT_FULL 1u
#define SLOT_TOMB 2u
#define SLOT_BUSY 3u
// states that exist only in DIFF LAYERS (views, see below): a removal marker (the key is absent in this view whatever the layers below hold) and
// an added entry that additionally hides an older entry of the same key in a lower layer (UtxoDiff: the outpoint is in `remove` AND in `add`)
#define SLOT_REMOVED 4u
#define SLOT_FULLH 5u
#define INLINE_SCRIPT 68u
#define SLOT_SCRIPT_BYTE 60u  // byte offset of the inline script inside the slot (word 15)

struct __align__(128) UtxoSlot {
  uint32_t state;
  uint32_t key[9];       // txid (8 words) + index
  uint64_t amount;       // word 10,11
  uint64_t daa;          // word 12,13
  uint32_t meta;         // spk_version | is_coinbase << 16 | script_len << 17
  uint8_t script[INLINE_SCRIPT];  // inline bytes, or (len > 68) a u64 offset into the overflow arena
};
static_assert(sizeof(UtxoSlot) == 128, "slot must be one 128-byte line");

struct kgv_utxo_table {
  UtxoSlot* slots = nullptr;
  uint64_t mask = 0;             // capacity - 1
  uint8_t* overflow = nullptr;   // long scripts (append-only between rehashes: offsets stay valid until kgv_utxo_rehash compacts the arena)
  uint64_t overflow_cap = 0;
  unsigned long long* counters = nullptr;  // [0] live entries, [1] tombstones, [2] overflow bytes used, [3] insert failures, [8..15] digest scratch
  // Composed views (consensus/core/src/utxo/utxo_view.rs:22-35: ComposedUtxoView = base view + UtxoDiff, nesting arbitrarily): a table with
  // base != nullptr is a DIFF LAYER over `base`; lookups probe it first and fall through, writes go to it and never touch what lies below.
  kgv_utxo_table* base = nullptr;
  struct TableView* d_view = nullptr;  // this table's TableView in device memory (what an upper layer's `below` points to)
  // maintenance (kgv_utxo_maint.cu)
  uint64_t rehashes = 0;
  uint32_t max_load = 0;         // growth policy in permille of the capacity, 0 = off
  uint64_t occ_bound = 0;        // with the policy on: upper bounds of the non-EMPTY slots and of counters[2] (exact at the last read + every
  uint64_t arena_bound = 0;      // write's reservation since), so that most writes need no counter read
  // the table's device and the order of the calls of every context on it (kgv_internal.h); shared with the contexts that still have
  // arrays of this table to release
  std::shared_ptr<struct kgv_table_sync> sync;
};

struct TableView {
  UtxoSlot* slots;
  uint64_t mask;
  uint8_t* overflow;
  uint64_t overflow_cap;
  unsigned long long* counters;
  const TableView* below;  // next lower layer of a composed view, nullptr for a plain table
};
static inline TableView view_of(const kgv_utxo_table* t) { return TableView{t->slots, t->mask, t->overflow, t->overflow_cap, t->counters, t->base ? t->base->d_view : nullptr}; }

namespace kgv {

// 32 bytes as two 128-bit accesses issued back to back (sm_90 has no 256-bit LDG / STG)
__device__ __forceinline__ void ld256_cg(uint32_t* w, const void* p) {
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.cg.v4.u32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
               : "l"(p)
               : "memory");
}
__device__ __forceinline__ void st256(void* p, const uint32_t* w) {
  asm volatile("st.global.v4.u32 [%8], {%0,%1,%2,%3};\n\t"
               "st.global.v4.u32 [%8+16], {%4,%5,%6,%7};" ::"r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "r"(w[4]), "r"(w[5]), "r"(w[6]),
               "r"(w[7]), "l"(p)
               : "memory");
}

// 36-byte outpoint (txid || index LE) -> 9 words.  Key arrays handed to the library are 4-byte aligned (36 * i keeps that).
__device__ __forceinline__ void load_key(uint32_t* k, const uint8_t* p) {
  if ((((uintptr_t)p) & 3) == 0) {
    const uint32_t* q = (const uint32_t*)p;
#pragma unroll
    for (int i = 0; i < 9; i++) k[i] = __ldg(q + i);
  } else {
#pragma unroll
    for (int i = 0; i < 9; i++) k[i] = (uint32_t)p[4 * i] | ((uint32_t)p[4 * i + 1] << 8) | ((uint32_t)p[4 * i + 2] << 16) | ((uint32_t)p[4 * i + 3] << 24);
  }
}
// key of a transaction input: prev_txid sits at the start of the 56-byte (8-byte aligned) kgv_input record
__device__ __forceinline__ void input_key(uint32_t* k, const kgv_input& in) {
  const uint32_t* q = (const uint32_t*)in.prev_txid;
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = q[w];
  k[8] = in.prev_index;
}
__device__ __forceinline__ uint64_t key_hash(const uint32_t* k) {
  // txids are BLAKE2b outputs (uniform); all nine words take part so crafted outpoints cannot pile up on a few slots
  uint64_t h = ((uint64_t)k[1] << 32 | k[0]) ^ (((uint64_t)k[3] << 32 | k[2]) * 0x9E3779B97F4A7C15ull);
  h ^= ((uint64_t)k[5] << 32 | k[4]) * 0xC2B2AE3D27D4EB4Full;
  h ^= ((uint64_t)k[7] << 32 | k[6]) * 0x165667B19E3779F9ull;
  h ^= (uint64_t)k[8] * 0xD6E8FEB86659FD93ull;
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 32;
  return h;
}
// first 64 bytes of a slot
struct SlotHead {
  uint32_t w[16];
  __device__ __forceinline__ uint32_t state() const { return w[0]; }
  __device__ __forceinline__ bool key_is(const uint32_t* k) const {
    bool eq = true;
#pragma unroll
    for (int i = 0; i < 9; i++) eq = eq && (w[1 + i] == k[i]);
    return eq;
  }
  __device__ __forceinline__ uint64_t amount() const { return (uint64_t)w[11] << 32 | w[10]; }
  __device__ __forceinline__ uint64_t daa() const { return (uint64_t)w[13] << 32 | w[12]; }
  __device__ __forceinline__ uint32_t meta() const { return w[14]; }
};
__device__ __forceinline__ void slot_load_head(SlotHead& h, const UtxoSlot* s) {
  ld256_cg(h.w, s);
  ld256_cg(h.w + 8, (const uint8_t*)s + 32);
}
// one layer: the slot holding key k in state FULL / FULLH / REMOVED (its first 64 bytes in `head`), or nullptr.  The table must not be
// modified concurrently by an operation on the SAME key.
__device__ __forceinline__ UtxoSlot* layer_find(const TableView& t, const uint32_t* k, SlotHead& head) {
  uint64_t i = key_hash(k) & t.mask;
  for (uint64_t probes = 0; probes <= t.mask; probes++) {
    UtxoSlot* s = &t.slots[i];
    slot_load_head(head, s);
    const uint32_t st = head.state();
    if (st == SLOT_EMPTY) return nullptr;
    if ((st == SLOT_FULL || st >= SLOT_REMOVED) && head.key_is(k)) return s;
    i = (i + 1) & t.mask;
  }
  return nullptr;
}
// UtxoView::get on the composed view: the first layer from the top that knows the key decides (added entry -> found, removal marker -> absent),
// utxo_view.rs:22-35.  *in_top (optional) tells whether the returned slot belongs to the top layer.
__device__ __forceinline__ UtxoSlot* table_find(const TableView& t, const uint32_t* k, SlotHead& head, bool* in_top = nullptr) {
  UtxoSlot* s = layer_find(t, k, head);
  if (in_top) *in_top = true;
  if (s) return head.state() == SLOT_REMOVED ? nullptr : s;
  if (in_top) *in_top = false;
  for (const TableView* L = t.below; L; L = L->below) {
    s = layer_find(*L, k, head);
    if (s) return head.state() == SLOT_REMOVED ? nullptr : s;
  }
  return nullptr;
}
// the layer of a composed view a slot belongs to (its overflow arena holds the slot's long script)
__device__ __forceinline__ const TableView* layer_of(const TableView& t, const UtxoSlot* s) {
  for (const TableView* L = &t; L; L = L->below)
    if (s >= L->slots && s <= L->slots + L->mask) return L;
  return &t;
}
__device__ __forceinline__ void head_to_entry(DevEntry& e, const TableView& t, const UtxoSlot* s, const SlotHead& h) {
  e.amount = h.amount();
  e.block_daa_score = h.daa();
  const uint32_t meta = h.meta();
  e.spk_version = (uint16_t)(meta & 0xFFFFu);
  e.is_coinbase = (uint8_t)((meta >> 16) & 1u);
  e.script_len = meta >> 17;
  if (e.script_len <= INLINE_SCRIPT) e.script = (const uint8_t*)s + SLOT_SCRIPT_BYTE;
  else {
    uint64_t off;
    memcpy(&off, s->script, 8);
    e.script = (t.below ? layer_of(t, s)->overflow : t.overflow) + off;
  }
  e.found = 1;
}
__device__ __forceinline__ void entry_absent(DevEntry& d) {
  d.amount = 0; d.block_daa_score = 0; d.script = nullptr; d.script_len = 0; d.spk_version = 0; d.is_coinbase = 0; d.found = 0;
}

// up to 68 script bytes at an arbitrarily aligned address -> 17 little-endian words (bytes past `len` are zero).
// Only aligned words that overlap [p, p+len) are read.
__device__ __forceinline__ void load_script_words(uint32_t* w, const uint8_t* p, uint32_t len) {
  const uint32_t mis = (uint32_t)((uintptr_t)p & 3);
  const uint32_t* q = (const uint32_t*)((uintptr_t)p - mis);
  const uint32_t sh = mis * 8;
  const uint32_t span = mis + len;                 // bytes from q[0] to the end of the script
  const uint32_t nq = (span + 3) >> 2;             // aligned words touched
  uint32_t prev = nq ? q[0] : 0u;
#pragma unroll
  for (int i = 0; i < 17; i++) {
    uint32_t nx = ((uint32_t)(i + 1) < nq) ? q[i + 1] : 0u;
    uint32_t v = __funnelshift_r(prev, nx, sh);
    const uint32_t have = (uint32_t)(4 * i) < len ? len - 4 * i : 0u;  // valid bytes in this word
    if (have < 4) v &= have ? (0xFFFFFFFFu >> (8 * (4 - have))) : 0u;
    w[i] = v;
    prev = nx;
  }
}

// upsert; returns 1 inserted, 2 replaced, 0 failed (table or overflow arena full).
// Keys inserted concurrently by one kernel must be distinct (API contract), so a slot another thread is
// filling (BUSY) always belongs to a different key and is simply skipped: no thread ever waits on another.
// In a diff layer (t.below != nullptr) the write goes to the top layer only: an added entry becomes FULLH when a lower layer (or a removal
// marker of this layer) holds the key, and `marker` = true stores a removal marker instead of an entry (UtxoDiff::remove_entry of an entry
// that lives below, utxo_diff.rs:249-258).
__device__ __forceinline__ uint32_t table_put(const TableView& t, const uint32_t* k, uint64_t amount, uint64_t daa, uint32_t spk_version, uint32_t is_coinbase,
                                              const uint8_t* script, uint32_t script_len, int* s_live = nullptr, int* s_tomb = nullptr, bool marker = false) {
  // s_live / s_tomb: optional shared-memory accumulators for the live / tombstone counters (the caller flushes them once per CTA)
  uint32_t final_state = marker ? SLOT_REMOVED : SLOT_FULL;
  if (t.below && !marker) {
    SlotHead hb;
    for (const TableView* L = t.below; L; L = L->below) {
      UtxoSlot* sb = layer_find(*L, k, hb);
      if (sb) { if (hb.state() != SLOT_REMOVED) final_state = SLOT_FULLH; break; }
    }
  }
  uint64_t i = key_hash(k) & t.mask;
  UtxoSlot* target = nullptr;
  UtxoSlot* tomb = nullptr;
  bool replace = false;
  SlotHead h;
  for (uint64_t probes = 0; probes <= t.mask; probes++, i = (i + 1) & t.mask) {
    UtxoSlot* s = &t.slots[i];
    slot_load_head(h, s);
    const uint32_t st = h.state();
    if (st == SLOT_FULL || st >= SLOT_REMOVED) {
      if (h.key_is(k)) {
        target = s; replace = true;
        if (st == SLOT_REMOVED && !marker) final_state = SLOT_FULLH;  // re-adding what this layer removed: the lower entry stays hidden
        if (st == SLOT_FULLH && !marker) final_state = SLOT_FULLH;
        break;
      }
      continue;
    }
    if (st == SLOT_TOMB) { if (!tomb) tomb = s; continue; }
    if (st == SLOT_BUSY) continue;
    // EMPTY: the key is not in the table. Prefer the first tombstone seen, else this slot.
    if (tomb) {
      if (atomicCAS(&tomb->state, SLOT_TOMB, SLOT_BUSY) == SLOT_TOMB) {
        target = tomb;
        if (s_tomb) atomicSub(s_tomb, 1); else atomicAdd(&t.counters[1], (unsigned long long)-1);
        break;
      }
      tomb = nullptr;
    }
    if (atomicCAS(&s->state, SLOT_EMPTY, SLOT_BUSY) == SLOT_EMPTY) { target = s; break; }
    // lost the race for this slot (it now holds another key): keep probing
  }
  if (!target && tomb && atomicCAS(&tomb->state, SLOT_TOMB, SLOT_BUSY) == SLOT_TOMB) {
    target = tomb;
    if (s_tomb) atomicSub(s_tomb, 1); else atomicAdd(&t.counters[1], (unsigned long long)-1);
  }
  if (!target) { atomicAdd(&t.counters[3], 1ull); return 0; }
  uint32_t w[32];
  w[0] = replace ? final_state : SLOT_BUSY;
#pragma unroll
  for (int j = 0; j < 9; j++) w[1 + j] = k[j];
  w[10] = (uint32_t)amount; w[11] = (uint32_t)(amount >> 32);
  w[12] = (uint32_t)daa; w[13] = (uint32_t)(daa >> 32);
  w[14] = (spk_version & 0xFFFFu) | ((is_coinbase & 1u) << 16) | (script_len << 17);
  if (script_len <= INLINE_SCRIPT) {
    load_script_words(w + 15, script, script_len);
  } else {
    uint64_t need = (script_len + 7u) & ~7ull;
    uint64_t off = atomicAdd(&t.counters[2], (unsigned long long)need);
    if (off + need > t.overflow_cap) {
      atomicAdd(&t.counters[3], 1ull);
      if (!replace) { __threadfence(); target->state = SLOT_TOMB; atomicAdd(&t.counters[1], 1ull); }
      return 0;
    }
    for (uint32_t b = 0; b < script_len; b++) t.overflow[off + b] = script[b];
    w[15] = (uint32_t)off; w[16] = (uint32_t)(off >> 32);
#pragma unroll
    for (int j = 17; j < 32; j++) w[j] = 0;
  }
  st256((uint8_t*)target + 32, w + 8);
  st256((uint8_t*)target + 64, w + 16);
  st256((uint8_t*)target + 96, w + 24);
  st256(target, w);
  if (!replace) {
    __threadfence();
    *(volatile uint32_t*)&target->state = final_state;
    if (s_live) atomicAdd(s_live, 1); else atomicAdd(&t.counters[0], 1ull);
  }
  return replace ? 2u : 1u;
}
// erase of an entry already located (slot s, found in the top layer or below): a plain table tombstones the slot; a diff layer turns its own
// added entry back into nothing (FULL) or into a removal marker (FULLH), and records a removal marker for an entry that lives below.
__device__ __forceinline__ void table_erase_found(const TableView& t, const uint32_t* k, UtxoSlot* s, bool in_top, int* s_live = nullptr, int* s_tomb = nullptr) {
  if (!in_top) {
    table_put(t, k, 0, 0, 0, 0, nullptr, 0, s_live, s_tomb, true);
    return;
  }
  const uint32_t st = *(volatile uint32_t*)&s->state;
  if (st == SLOT_FULLH) { *(volatile uint32_t*)&s->state = SLOT_REMOVED; return; }  // still one entry of this layer (now a marker)
  *(volatile uint32_t*)&s->state = SLOT_TOMB;
  if (s_live) { atomicSub(s_live, 1); atomicAdd(s_tomb, 1); }
  else { atomicAdd(&t.counters[0], (unsigned long long)-1); atomicAdd(&t.counters[1], 1ull); }
}
__device__ __forceinline__ uint32_t table_erase(const TableView& t, const uint32_t* k) {
  SlotHead h;
  bool in_top;
  UtxoSlot* s = table_find(t, k, h, &in_top);
  if (!s) return 0;
  table_erase_found(t, k, s, in_top);
  return 1;
}

}  // namespace kgv
