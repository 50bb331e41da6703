// Host build of the coinbase side of kgv_replay_verify_chain (kgv_chain.cuh) for GPU-less tests (TEST BUILD ONLY): the payload parser and
// expected_coinbase_hash, the same functions k_chain_blocks / k_chain_verdict call.
#include "../../rusty_kaspa_b200/csrc/kgv_chain.cuh"
using namespace kgv;

extern "C" {
// deserialize_coinbase_payload: 0 or the KGV_COINBASE_PAYLOAD_* code
uint32_t hs_payload_parse(const uint8_t* payload, uint32_t len, uint64_t max_payload_len, uint64_t max_spk_len) {
  CoinbasePayload c;
  uint64_t a, b;
  return coinbase_payload_parse(c, payload, len, max_payload_len, max_spk_len, a, b);
}
// The expected coinbase of a mergeset of n blocks (block j: subsidy[j], fees[j], flags[j] KGV_MERGED_*, script arena[off[j] .. +len[j]] of
// version ver[j]) for a chain block whose own payload is miner_payload: returns KGV_CHAIN_OK with the tx hash in out32,
// KGV_CHAIN_COINBASE_PAYLOAD_UNPARSABLE or KGV_CHAIN_REWARD_OVERFLOW, as k_chain_verdict decides check 4.
uint32_t hs_expected_coinbase(uint32_t n, const uint64_t* subsidy, const uint64_t* fees, const uint8_t* flags, const uint8_t* arena, const uint32_t* off,
                              const uint32_t* len, const uint16_t* ver, uint64_t blue_score, uint64_t expected_subsidy, const uint8_t* miner_payload,
                              uint32_t miner_len, uint64_t max_payload_len, uint64_t max_spk_len, uint8_t* out32) {
  CoinbasePayload miner;
  uint64_t a, b;
  if (coinbase_payload_parse(miner, miner_payload, miner_len, max_payload_len, max_spk_len, a, b)) return KGV_CHAIN_COINBASE_PAYLOAD_UNPARSABLE;
  auto rw = [&](uint32_t j) {
    MergedReward r;
    r.subsidy = subsidy[j]; r.fees = fees[j]; r.script = arena + off[j]; r.script_len = len[j]; r.spk_version = ver[j]; r.flags = flags[j];
    return r;
  };
  uint64_t d[4];
  if (!expected_coinbase_hash(d, n, rw, blue_score, expected_subsidy, miner_payload, miner_len, miner)) return KGV_CHAIN_REWARD_OVERFLOW;
  for (int k = 0; k < 32; k++) out32[k] = (uint8_t)(d[k / 8] >> (8 * (k % 8)));
  return KGV_CHAIN_OK;
}
}
