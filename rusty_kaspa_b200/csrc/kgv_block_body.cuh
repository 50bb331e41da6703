// kgv_block_body.cuh — device pieces of the block body rules (kgv_block_body.cu): the hashed sets behind the three set checks, the
// saturating mass triple of check_block_mass and the coinbase payload rule.
//
// Restates, in the reference's check order:
//   check_block_mass / check_duplicate_transactions / check_block_double_spends / check_no_chained_transactions
//                                          consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:63-131
//   check_coinbase_blue_score_and_subsidy  body_validation_in_context.rs:63-80
#pragma once
#include "kgv_chain.cuh"

namespace kgv {

constexpr uint32_t BODY_NONE = 0xFFFFFFFFu;        // no offender / empty set slot

// ---- open-addressed sets of item indices ----
// A set has cap >= 2 * (items inserted) slots, so a probe walk always meets an empty slot.  A slot holds the LOWEST index among the inserted
// items of one key (HashSet::insert returns false for every later one).  eq(j) tells whether item j has the key being inserted / looked up;
// once a slot is taken every value it ever holds is an item of that one key, so comparing against any snapshot of it is exact.
__device__ __forceinline__ uint64_t body_mix(uint64_t h) {  // murmur3's finalizer, a bijection of the state
  h ^= h >> 33; h *= 0xFF51AFD7ED558CCDull; h ^= h >> 33; h *= 0xC4CEB9FE1A85EC53ull; h ^= h >> 33;
  return h;
}
// Keyed hashes of the 32-byte id and of the 36-byte outpoint.  The secret salt is the initial state and every 64-bit word of the key is
// xored into the state before it is mixed again, so whether two keys meet depends on the salt at every word: a peer who chooses the
// outpoints (nothing has looked them up yet) cannot compute a set of keys that share a slot, and probe runs stay short for any body.
__device__ __forceinline__ uint64_t body_hash_id(const uint64_t* id, uint64_t salt) {
  uint64_t h = salt;
#pragma unroll
  for (int k = 0; k < 4; k++) h = body_mix(h ^ id[k]);
  return h;
}
__device__ __forceinline__ uint64_t body_hash_outpoint(const kgv_input& in, uint64_t salt) {
  return body_mix(body_hash_id(reinterpret_cast<const uint64_t*>(in.prev_txid), salt) ^ in.prev_index);  // prev_txid is 8-byte aligned
}
__device__ __forceinline__ uint32_t body_slot(uint64_t h, uint32_t cap) { return (uint32_t)(((h >> 32) * cap) >> 32); }

template <class Eq>
__device__ __forceinline__ void body_set_insert(uint32_t* tab, uint32_t cap, uint64_t h, uint32_t item, Eq eq) {
  for (uint32_t s = body_slot(h, cap);; s = s + 1 == cap ? 0 : s + 1) {
    const uint32_t cur = atomicCAS(&tab[s], BODY_NONE, item);
    if (cur == BODY_NONE) return;
    if (eq(cur)) { atomicMin(&tab[s], item); return; }
  }
}
// lowest inserted item with the key, BODY_NONE if there is none (call after every insert is done)
template <class Eq>
__device__ __forceinline__ uint32_t body_set_find(const uint32_t* tab, uint32_t cap, uint64_t h, Eq eq) {
  for (uint32_t s = body_slot(h, cap);; s = s + 1 == cap ? 0 : s + 1) {
    const uint32_t cur = tab[s];
    if (cur == BODY_NONE || eq(cur)) return cur;
  }
}

__device__ __forceinline__ bool body_same_id(const uint64_t* a, const uint64_t* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2] && a[3] == b[3]; }
__device__ __forceinline__ bool body_same_outpoint(const kgv_input& a, const kgv_input& b) {
  const uint64_t* x = reinterpret_cast<const uint64_t*>(a.prev_txid);  // 8-byte aligned: kgv_input is 56 bytes, prev_txid first
  const uint64_t* y = reinterpret_cast<const uint64_t*>(b.prev_txid);
  return a.prev_index == b.prev_index && body_same_id(x, y);
}

// ---- check_block_mass: the three running totals, each a saturating sum (associative over u64, so they scan) ----
struct BodyMass { uint64_t compute, transient, storage; };
__device__ __forceinline__ uint64_t body_sat_add(uint64_t a, uint64_t b) { return a + b < a ? ~0ull : a + b; }
struct BodyMassAdd {
  __device__ __forceinline__ BodyMass operator()(const BodyMass& a, const BodyMass& b) const {
    return BodyMass{body_sat_add(a.compute, b.compute), body_sat_add(a.transient, b.transient), body_sat_add(a.storage, b.storage)};
  }
};

// ---- check_coinbase_blue_score_and_subsidy on the coinbase's payload (parsed by coinbase_payload_parse, kgv_chain.cuh) ----
__device__ __forceinline__ void body_coinbase_payload(kgv_body_result& r, const uint8_t* payload, uint32_t len, const kgv_block_header_ctx& h, uint64_t max_payload_len,
                                                      uint64_t max_spk_len) {
  CoinbasePayload c;
  uint64_t a = 0, b = 0;
  const uint32_t e = coinbase_payload_parse(c, payload, len, max_payload_len, max_spk_len, a, b);
  if (e) { r.status = KGV_BODY_BAD_COINBASE_PAYLOAD; r.tx_status = e; r.a = a; r.b = b; return; }
  if (c.blue_score != h.blue_score) { r.status = KGV_BODY_BAD_COINBASE_PAYLOAD_BLUE_SCORE; r.a = c.blue_score; r.b = h.blue_score; return; }
  if (c.subsidy != h.expected_subsidy) { r.status = KGV_BODY_WRONG_SUBSIDY; r.a = h.expected_subsidy; r.b = c.subsidy; }
}

}  // namespace kgv
