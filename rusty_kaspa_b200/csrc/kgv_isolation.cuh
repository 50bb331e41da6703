// kgv_isolation.cuh — the per-transaction rules that need no UTXO context, one warp per transaction.
//
// Restates, in the reference's check order:
//   validate_tx_in_isolation            consensus/src/processes/transaction_validator/tx_validation_in_isolation.rs:16-26
//   check_tx_is_finalized               tx_validation_in_header_context.rs (validate_tx_in_header_context_with_args)
//   calc_non_contextual_masses          consensus/core/src/mass/mod.rs:248-269, transaction_estimated_serialized_size :13-59
// Every "first offender" is the lowest index, as the reference's `position` / enumerate loops find it.  The warp strides over a
// transaction's inputs and outputs 32 at a time; duplicate inputs are compared pairwise through shuffles up to 32 inputs, larger
// transactions go to a block-wide sort (k_tx_isolation_large in kgv_isolation.cu).
#pragma once
#include "kgv_txhash.cuh"
#include "kgv_utxo.cuh"

namespace kgv {

constexpr uint64_t ISO_MAX_SOMPI = 29000000000ull * 100000000ull;  // constants::MAX_SOMPI
constexpr uint64_t ISO_LOCK_TIME_THRESHOLD = 500000000000ull;      // constants::LOCK_TIME_THRESHOLD
constexpr uint64_t ISO_TRANSIENT_BYTE_TO_MASS_FACTOR = 4;          // constants::TRANSIENT_BYTE_TO_MASS_FACTOR
constexpr uint16_t ISO_TX_VERSION = 0;                             // constants::TX_VERSION
constexpr uint32_t ISO_WARP_DUP_MAX = 32;                          // inputs a warp checks for duplicates by itself
constexpr unsigned ISO_FULL = 0xFFFFFFFFu;

// the header context the finality rule reads for transaction ti: one pair for the whole batch, or (headers != null) the values of the
// transaction's own block
struct IsoContext {
  uint64_t daa_score, past_median_time;
  const kgv_block_header_ctx* headers;
  const uint32_t* tx_block;
  __device__ __forceinline__ uint64_t daa(uint32_t ti) const { return headers ? headers[tx_block[ti]].daa_score : daa_score; }
  __device__ __forceinline__ uint64_t pmt(uint32_t ti) const { return headers ? headers[tx_block[ti]].past_median_time : past_median_time; }
};

// first index in [0, n) where pred holds, n if none; n must be the same on every lane, and every lane returns the answer
template <class P>
__device__ __forceinline__ uint32_t warp_first(uint32_t n, uint32_t lane, P pred) {
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t i = base + lane;
    const unsigned m = __ballot_sync(ISO_FULL, i < n && pred(i));
    if (m) return base + __ffs(m) - 1;
  }
  return n;
}

__device__ __forceinline__ uint64_t warp_sum(uint64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(ISO_FULL, v, o);
  return v;
}

__device__ __forceinline__ kgv_tx_result iso_result(uint8_t status, uint32_t index) {
  kgv_tx_result r;
  r.fee = 0; r.fail_input = index; r.status = status; r.script_err = 0; r.pad_[0] = r.pad_[1] = 0;
  return r;
}

// calc_non_contextual_masses in wrapping u64 arithmetic (a release build of the reference); (0, 0) for a coinbase
__device__ __forceinline__ kgv_tx_masses iso_masses(const BatchView& b, const kgv_tx& t, bool cb, const kgv_tx_rules& r, uint32_t lane) {
  uint64_t in_bytes = 0, sigops = 0, out_bytes = 0, spk_bytes = 0;
  for (uint32_t i = lane; i < t.n_inputs; i += 32) {
    const kgv_input& in = b.inputs[t.first_input + i];
    in_bytes += 32 + 4 + 8 + (uint64_t)in.sigscript_len + 8;  // outpoint, script length, script, sequence
    sigops += in.sig_op_count;
  }
  for (uint32_t i = lane; i < t.n_outputs; i += 32) {
    const uint64_t l = b.outputs[t.first_output + i].script_len;
    out_bytes += 8 + 2 + 8 + l;  // value, spk version, script length, script
    spk_bytes += 2 + l;
  }
  in_bytes = warp_sum(in_bytes); sigops = warp_sum(sigops); out_bytes = warp_sum(out_bytes); spk_bytes = warp_sum(spk_bytes);
  kgv_tx_masses m;
  m.compute_mass = m.transient_mass = 0;
  if (cb) return m;
  // version, input count, inputs, output count, outputs, lock time, subnetwork id, gas, payload hash, payload length, payload
  const uint64_t size = 2 + 8 + in_bytes + 8 + out_bytes + 8 + 20 + 8 + 32 + 8 + (uint64_t)t.payload_len;
  m.compute_mass = size * r.mass_per_tx_byte + spk_bytes * r.mass_per_script_pub_key_byte + sigops * r.mass_per_sig_op;
  m.transient_mass = size * ISO_TRANSIENT_BYTE_TO_MASS_FACTOR;
  return m;
}

// check_transaction_output_value_ranges: the outputs in order, each checked for zero, for > MAX_SOMPI, then added to the running total
// (overflow, then > MAX_SOMPI).  The warp scans 32 values at a time with a saturating sum; the first lane where anything fails decides.
__device__ __forceinline__ kgv_tx_result iso_output_values(const BatchView& b, const kgv_tx& t, uint32_t lane) {
  uint64_t carry = 0;  // total of the outputs before this chunk (<= MAX_SOMPI, else the loop has returned)
  for (uint32_t base = 0; base < t.n_outputs; base += 32) {
    const uint32_t i = base + lane;
    const uint64_t v = i < t.n_outputs ? b.outputs[t.first_output + i].value : 0;
    uint64_t s = v;  // saturating inclusive prefix within the chunk
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t u = __shfl_up_sync(ISO_FULL, s, o);
      if (lane >= (uint32_t)o) s = s + u < s ? ~0ull : s + u;
    }
    const uint64_t tot = carry + s < carry ? ~0ull : carry + s;
    const bool bad = i < t.n_outputs && (v == 0 || v > ISO_MAX_SOMPI || tot > ISO_MAX_SOMPI);
    const unsigned m = __ballot_sync(ISO_FULL, bad);
    if (m) {
      const int j = __ffs(m) - 1;
      const uint64_t vj = __shfl_sync(ISO_FULL, v, j), tj = __shfl_sync(ISO_FULL, tot, j);
      if (vj == 0) return iso_result(KGV_TX_TX_OUT_ZERO, base + j);
      if (vj > ISO_MAX_SOMPI) return iso_result(KGV_TX_TX_OUT_TOO_HIGH, base + j);
      // every earlier value and the total before j are <= MAX_SOMPI, so tj = before + vj is exact
      uint64_t before = tj - vj, total;
      if (ck_add(before, vj, total)) return iso_result(KGV_TX_OUTPUTS_VALUE_OVERFLOW, 0);
      return iso_result(KGV_TX_TOTAL_TX_OUT_TOO_HIGH, 0);
    }
    carry = __shfl_sync(ISO_FULL, tot, 31);
  }
  return iso_result(KGV_TX_OK, 0);
}

// check_duplicate_transaction_inputs for at most 32 inputs: lane i holds outpoint i; each earlier outpoint is broadcast by its 64-bit
// hash and, only when some later lane has the same hash, word by word for the exact comparison
__device__ __forceinline__ bool iso_warp_duplicates(const BatchView& b, const kgv_tx& t, uint32_t lane) {
  const uint32_t n = t.n_inputs;
  uint32_t k[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  uint64_t h = 0;
  if (lane < n) { input_key(k, b.inputs[t.first_input + lane]); h = key_hash(k); }
  bool dup = false;
  for (uint32_t j = 0; j + 1 < n; j++) {
    const uint64_t hj = __shfl_sync(ISO_FULL, h, j);
    bool eq = lane > j && lane < n && h == hj;
    if (__any_sync(ISO_FULL, eq)) {
#pragma unroll
      for (int w = 0; w < 9; w++) eq = (__shfl_sync(ISO_FULL, k[w], j) == k[w]) && eq;
      dup = dup || eq;
    }
  }
  return __any_sync(ISO_FULL, dup);
}

// the checks after the duplicate-input check: check_gas, check_transaction_subnetwork, check_transaction_version, then finality
__device__ __forceinline__ kgv_tx_result iso_tail(const BatchView& b, const kgv_tx& t, bool cb, uint64_t daa, uint64_t pmt, bool finality, uint32_t lane) {
  if (t.gas > 0) return iso_result(KGV_TX_HAS_GAS, 0);
  if (!cb && !tx_is_native(t)) return iso_result(KGV_TX_SUBNETWORKS_DISABLED, 0);
  if (t.version != ISO_TX_VERSION) return iso_result(KGV_TX_UNKNOWN_TX_VERSION, 0);
  if (!finality || t.lock_time == 0) return iso_result(KGV_TX_OK, 0);
  const uint64_t ref = t.lock_time < ISO_LOCK_TIME_THRESHOLD ? daa : pmt;
  if (t.lock_time < ref) return iso_result(KGV_TX_OK, 0);
  const kgv_input* in = b.inputs + t.first_input;
  const uint32_t i = warp_first(t.n_inputs, lane, [&](uint32_t x) { return in[x].sequence != ~0ull; });
  return i < t.n_inputs ? iso_result(KGV_TX_NOT_FINALIZED, i) : iso_result(KGV_TX_OK, 0);
}

// validate_tx_in_isolation up to (not including) the duplicate-input check
__device__ __forceinline__ kgv_tx_result iso_head(const BatchView& b, const kgv_tx& t, bool cb, const kgv_tx_rules& r, uint32_t lane) {
  // check_transaction_inputs_count, check_transaction_signature_scripts
  if (!cb && t.n_inputs == 0) return iso_result(KGV_TX_NO_TX_INPUTS, 0);
  if (t.n_inputs > r.max_tx_inputs) return iso_result(KGV_TX_TOO_MANY_INPUTS, 0);
  const kgv_input* in = b.inputs + t.first_input;
  const kgv_output* out = b.outputs + t.first_output;
  uint32_t i = warp_first(t.n_inputs, lane, [&](uint32_t x) { return in[x].sigscript_len > r.max_signature_script_len; });
  if (i < t.n_inputs) return iso_result(KGV_TX_TOO_BIG_SIGNATURE_SCRIPT, i);
  // check_transaction_outputs_count (skipped for a coinbase), check_transaction_script_public_keys
  if (!cb && t.n_outputs > r.max_tx_outputs) return iso_result(KGV_TX_TOO_MANY_OUTPUTS, 0);
  i = warp_first(t.n_outputs, lane, [&](uint32_t x) { return out[x].script_len > r.max_script_public_key_len; });
  if (i < t.n_outputs) return iso_result(KGV_TX_TOO_BIG_SCRIPT_PUBLIC_KEY, i);
  // check_coinbase_in_isolation
  if (cb) {
    if (t.n_inputs) return iso_result(KGV_TX_COINBASE_HAS_INPUTS, 0);
    if (t.mass > 0) return iso_result(KGV_TX_COINBASE_NON_ZERO_MASS_COMMITMENT, 0);
    if ((uint64_t)t.n_outputs > r.ghostdag_k + 2) return iso_result(KGV_TX_COINBASE_TOO_MANY_OUTPUTS, 0);
    i = warp_first(t.n_outputs, lane, [&](uint32_t x) { return out[x].script_len > r.coinbase_payload_script_public_key_max_len; });
    if (i < t.n_outputs) return iso_result(KGV_TX_COINBASE_SCRIPT_PUBLIC_KEY_TOO_LONG, i);
  }
  return iso_output_values(b, t, lane);
}

}  // namespace kgv
