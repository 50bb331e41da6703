// kgv_context.cuh — the UTXO-context rules of one transaction (K6), shared by the batch kernel (k_tx_context) and the
// in-order replay kernel.  Follows validate_populated_transaction_and_get_fee
// (consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs:34-61): coinbase maturity :75-91,
// input amounts :93-108, output amounts / fee :110-118, storage mass :120-128, sequence locks :130-155; the populate step
// that precedes it (first missing entry => MissingTxOutpoints) is utxo_validation.rs:319-327.
// The mempool form (mempool_context_rules) runs the same rule bodies in the order of validate_mempool_transaction_in_utxo_context
// (utxo_validation.rs:370-397) and adds the feerate threshold (tx_validation_in_utxo_context.rs:50-52,63-73).
#pragma once
#include "kgv_txhash.cuh"

namespace kgv {

// ---- the rule bodies: each returns KGV_TX_OK or the status of the rule that failed
__device__ __forceinline__ uint8_t rule_missing(const DevEntry* ent, uint32_t n_in) {
  for (uint32_t i = 0; i < n_in; i++)
    if (!ent[i].found) return KGV_TX_MISSING_OUTPOINTS;
  return KGV_TX_OK;
}
__device__ __forceinline__ uint8_t rule_maturity(const DevEntry* ent, uint32_t n_in, uint64_t pov, const kgv_params& prm, uint32_t& fail_input) {
  for (uint32_t i = 0; i < n_in; i++)
    if (ent[i].is_coinbase && ent[i].block_daa_score + prm.coinbase_maturity > pov) { fail_input = i; return KGV_TX_IMMATURE_COINBASE; }
  return KGV_TX_OK;
}
// input amounts and output values; the fee is written when both pass
__device__ __forceinline__ uint8_t rule_amounts(const BatchView& b, const kgv_tx& t, const DevEntry* ent, const kgv_params& prm, uint64_t& fee) {
  uint64_t total_in = 0;
  for (uint32_t i = 0; i < t.n_inputs; i++) {
    if (ck_add(total_in, ent[i].amount, total_in)) return KGV_TX_INPUT_AMOUNT_OVERFLOW;
    if (total_in > prm.max_sompi) return KGV_TX_INPUT_AMOUNT_TOO_HIGH;
  }
  uint64_t total_out = 0;
  for (uint32_t i = 0; i < t.n_outputs; i++) total_out += b.outputs[t.first_output + i].value;
  if (total_in < total_out) return KGV_TX_SPEND_TOO_HIGH;
  fee = total_in - total_out;
  return KGV_TX_OK;
}
// calc_contextual_masses(..).storage_mass; false: MassIncomputable
__device__ __forceinline__ bool tx_storage_mass(const BatchView& b, const kgv_tx& t, const DevEntry* ent, const kgv_params& prm, uint64_t& mass) {
  const kgv_output* outs = b.outputs + t.first_output;
  return storage_mass(mass, false, t.n_inputs, t.n_outputs, [&](uint32_t i) -> const DevEntry& { return ent[i]; },
                      [&](uint32_t i, uint64_t& v, uint32_t& l) { v = outs[i].value; l = outs[i].script_len; }, prm.storage_mass_parameter);
}
__device__ __forceinline__ uint8_t rule_sequence_lock(const BatchView& b, const kgv_tx& t, const DevEntry* ent, uint64_t pov) {
  for (uint32_t i = 0; i < t.n_inputs; i++) {
    uint64_t seq = b.inputs[t.first_input + i].sequence;
    if (seq & (1ull << 63)) continue;
    long long lock = (long long)ent[i].block_daa_score + (long long)(seq & 0xFFFFFFFFull) - 1;
    if (lock >= (long long)pov) return KGV_TX_SEQUENCE_LOCK;
  }
  return KGV_TX_OK;
}

__device__ __forceinline__ kgv_tx_result result_ok() {
  kgv_tx_result r;
  r.fee = 0; r.fail_input = 0; r.status = KGV_TX_OK; r.script_err = 0; r.pad_[0] = r.pad_[1] = 0;
  return r;
}

// b.entries must hold one DevEntry per input.  `skip` marks the transaction as a coinbase to be skipped
// (utxo_validation.rs:273 skips position 0; the batch kernels recognise it by its subnetwork id).
__device__ __forceinline__ kgv_tx_result tx_context_rules(const BatchView& b, uint32_t ti, uint64_t pov, uint32_t flags, const kgv_params& prm, bool skip) {
  const kgv_tx& t = b.txs[ti];
  kgv_tx_result r = result_ok();
  const DevEntry* ent = b.entries + t.first_input;
  if (skip) { r.status = KGV_TX_SKIPPED_COINBASE; return r; }
  if ((r.status = rule_missing(ent, t.n_inputs)) != KGV_TX_OK) return r;  // utxo_validation.rs:319-327
  if (flags == KGV_FLAGS_SCRIPTS_ONLY) return r;
  if ((r.status = rule_maturity(ent, t.n_inputs, pov, prm, r.fail_input)) != KGV_TX_OK) return r;
  if ((r.status = rule_amounts(b, t, ent, prm, r.fee)) != KGV_TX_OK) return r;
  if (flags != KGV_FLAGS_SKIP_MASS_CHECK) {
    uint64_t mass;
    if (!tx_storage_mass(b, t, ent, prm, mass)) { r.status = KGV_TX_MASS_INCOMPUTABLE; return r; }
    if (mass != t.mass) { r.status = KGV_TX_WRONG_MASS; return r; }
  }
  r.status = rule_sequence_lock(b, t, ent, pov);
  return r;
}

// validate_mempool_transaction_in_utxo_context (utxo_validation.rs:370-397) up to the scripts: missing -> storage mass
// (computed, never compared with the committed one: SkipMassCheck) -> maturity -> amounts -> sequence lock -> feerate.
// `mass` receives the storage mass once it is computed (0 before).  threshold NaN: no feerate check; otherwise
// fee / max(storage mass, nc_mass) <= threshold is FeerateTooLow, in f64 with round-to-nearest conversions and division as
// Rust's `as f64` and `/`.  A zero divisor sets `bad_threshold` (the reference asserts it is not zero).
__device__ __forceinline__ kgv_tx_result mempool_context_rules(const BatchView& b, uint32_t ti, uint64_t pov, const kgv_params& prm, double threshold,
                                                               uint64_t nc_mass, uint64_t& mass, bool& bad_threshold) {
  const kgv_tx& t = b.txs[ti];
  kgv_tx_result r = result_ok();
  const DevEntry* ent = b.entries + t.first_input;
  mass = 0;
  bad_threshold = false;
  if (tx_is_coinbase(t)) { r.status = KGV_TX_SKIPPED_COINBASE; return r; }
  if ((r.status = rule_missing(ent, t.n_inputs)) != KGV_TX_OK) return r;
  if (!tx_storage_mass(b, t, ent, prm, mass)) { r.status = KGV_TX_MASS_INCOMPUTABLE; return r; }
  if ((r.status = rule_maturity(ent, t.n_inputs, pov, prm, r.fail_input)) != KGV_TX_OK) return r;
  if ((r.status = rule_amounts(b, t, ent, prm, r.fee)) != KGV_TX_OK) return r;
  if ((r.status = rule_sequence_lock(b, t, ent, pov)) != KGV_TX_OK) return r;
  if (threshold == threshold) {  // not NaN
    const uint64_t m = mass > nc_mass ? mass : nc_mass;
    if (m == 0) { bad_threshold = true; return r; }
    if (__ddiv_rn(__ull2double_rn(r.fee), __ull2double_rn(m)) <= threshold) r.status = KGV_TX_FEERATE_TOO_LOW;
  }
  return r;
}

}  // namespace kgv
