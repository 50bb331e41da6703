// kgv_chain.cuh — the coinbase side of a chain block's UTXO state (kgv_replay_verify_chain, kgv_chain.cu): the coinbase payload parser
// the body rules share, and the expected coinbase streamed through the transaction-hash BLAKE2b.
//
// Restates:
//   deserialize_coinbase_payload     consensus/src/processes/coinbase.rs:185-220
//   expected_coinbase_transaction    coinbase.rs:97-142 (with serialize_coinbase_payload, :144-161)
//   hashing::tx::hash                consensus/core/src/hashing/tx.rs:45-107 (write_transaction, FULL)
// Host-compilable (KGV_HD): tests/hostsim/hostsim_chain.cpp builds the same functions with g++.
#pragma once
#include "kgv_txhash.cuh"

namespace kgv {

constexpr uint32_t COINBASE_MIN_PAYLOAD_LENGTH = 19;  // coinbase.rs MIN_PAYLOAD_LENGTH: blue score 8, subsidy 8, spk version 2, spk length 1

KGV_HD uint64_t le64(const uint8_t* p) {
  uint64_t v = 0;
  for (int i = 7; i >= 0; i--) v = v << 8 | p[i];
  return v;
}

// CoinbaseData of a payload; the script is at payload + 19, the extra data follows it
struct CoinbasePayload {
  uint64_t blue_score, subsidy;
  uint32_t spk_version, spk_len;
};
// deserialize_coinbase_payload: 0, or the KGV_COINBASE_PAYLOAD_* code with the CoinbaseError's two numbers in a, b.  Lengths are compared
// before any byte is read.
KGV_HD uint32_t coinbase_payload_parse(CoinbasePayload& c, const uint8_t* payload, uint32_t len, uint64_t max_payload_len, uint64_t max_spk_len, uint64_t& a,
                                       uint64_t& b) {
  if (len < COINBASE_MIN_PAYLOAD_LENGTH) { a = len; b = COINBASE_MIN_PAYLOAD_LENGTH; return KGV_COINBASE_PAYLOAD_LEN_BELOW_MIN; }
  if (len > max_payload_len) { a = len; b = max_payload_len; return KGV_COINBASE_PAYLOAD_LEN_ABOVE_MAX; }
  c.blue_score = le64(payload);
  c.subsidy = le64(payload + 8);
  c.spk_version = (uint32_t)payload[16] | (uint32_t)payload[17] << 8;
  c.spk_len = payload[18];
  if (c.spk_len > max_spk_len) { a = c.spk_len; b = max_spk_len; return KGV_COINBASE_PAYLOAD_SPK_LEN_ABOVE_MAX; }
  if (len - COINBASE_MIN_PAYLOAD_LENGTH < c.spk_len) { a = len; b = COINBASE_MIN_PAYLOAD_LENGTH + c.spk_len; return KGV_COINBASE_PAYLOAD_CANT_CONTAIN_SPK; }
  return 0;
}

// One entry of mergeset_rewards (BlockRewardData: the merged block's own payload subsidy and script, the fees of its accepted transactions)
// and its GHOSTDAG class (KGV_MERGED_*).
struct MergedReward {
  uint64_t subsidy, fees;
  const uint8_t* script;
  uint32_t script_len, spk_version, flags;
};

KGV_HD bool add_u64(uint64_t& acc, uint64_t v) {  // false where the reference's checked addition panics
  const uint64_t s = acc + v;
  if (s < acc) return false;
  acc = s;
  return true;
}

// hashing::tx::hash of expected_coinbase_transaction(daa_score, miner_data, ghostdag_data, mergeset_rewards, mergeset_non_daa) for a mergeset
// of n blocks in group order (selected parent first; restricted to the blues that is mergeset_blues order).  rw(j) gives block j's
// MergedReward.  miner_payload is the chain block's own coinbase payload, already parsed: the expected payload is its blue score and subsidy
// replaced by blue_score / expected_subsidy, the rest (script version, length, script, extra data) kept byte for byte.  Returns false where
// the reference panics on an overflow (subsidy + total_fees of a rewarded blue, a red's reward, the red sum); out4 is then untouched.
// Two passes over the rewards: the output count precedes the outputs in the encoding.  No dynamically indexed array but the hasher's.
template <class Rewards>
KGV_HD bool expected_coinbase_hash(uint64_t* out4, uint32_t n, Rewards rw, uint64_t blue_score, uint64_t expected_subsidy, const uint8_t* miner_payload,
                                   uint32_t miner_payload_len, const CoinbasePayload& miner) {
  uint64_t n_out = 0, red = 0;
  for (uint32_t j = 0; j < n; j++) {
    const MergedReward r = rw(j);
    if (r.flags & KGV_MERGED_RED) {
      uint64_t v = r.fees;
      if (!(r.flags & KGV_MERGED_NON_DAA) && !add_u64(v, r.subsidy)) return false;
      if (!add_u64(red, v)) return false;
    } else if (!(r.flags & KGV_MERGED_NON_DAA)) {
      uint64_t v = r.subsidy;
      if (!add_u64(v, r.fees)) return false;
      n_out += v > 0;
    }
  }
  n_out += red > 0;
  Blake2b s;
  b2b_init(s, B2B_TX_HASH);
  b2b_u16(s, 0);  // TX_VERSION
  b2b_u64(s, 0);  // no inputs
  b2b_u64(s, n_out);
  for (uint32_t j = 0; j < n; j++) {
    const MergedReward r = rw(j);
    if (r.flags & (KGV_MERGED_RED | KGV_MERGED_NON_DAA)) continue;
    const uint64_t v = r.subsidy + r.fees;  // checked in the first pass
    if (v == 0) continue;
    b2b_u64(s, v);
    b2b_u16(s, r.spk_version);
    b2b_var_bytes(s, r.script, r.script_len);
  }
  if (red > 0) {  // paid to the chain block's miner script
    b2b_u64(s, red);
    b2b_u16(s, miner.spk_version);
    b2b_var_bytes(s, miner_payload + COINBASE_MIN_PAYLOAD_LENGTH, miner.spk_len);
  }
  b2b_u64(s, 0);  // lock time
  b2b_u8(s, 1);   // SUBNETWORK_ID_COINBASE = 01 00 .. 00
  for (int i = 1; i < 20; i++) b2b_u8(s, 0);
  b2b_u64(s, 0);  // gas
  b2b_u64(s, miner_payload_len);
  b2b_u64(s, blue_score);
  b2b_u64(s, expected_subsidy);
  b2b_bytes(s, miner_payload + 16, miner_payload_len - 16);
  // mass 0: not written
  b2b_final(s, out4);
  return true;
}

}  // namespace kgv
