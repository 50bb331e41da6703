// kgv.hpp — C++17 host-side mirror of the reference interface for the validation hot path, on top of the C ABI (kgv.h).
//
// The reference is Rust; no Rust toolchain exists in the build image, so the typed host layer a Rust shim would provide
// is written in C++ (header only, RAII, exceptions for transport errors).  Names and argument meaning follow the
// reference so that call sites read like the original:
//   kgv::Transaction / TransactionInput / TransactionOutput / UtxoEntry     consensus/core/src/tx.rs:49-185
//   kgv::TransactionValidator::validate_populated_transaction_and_get_fee*  consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs:34-61
//   kgv::TransactionValidator::validate_transactions_in_parallel           consensus/src/pipeline/virtual_processor/utxo_validation.rs:262-278
//   kgv::TransactionValidator::validate_transactions_with_muhash_in_parallel  …:282-309
//   kgv::UtxoSet (get / write_diff / add_transactions)                      consensus/src/model/stores/utxo_set.rs:107-112, consensus/core/src/utxo/utxo_diff.rs:233-247
//   kgv::MuHash (add_element / remove_element / combine / finalize / serialize)  crypto/muhash/src/lib.rs:59-121
//   kgv::SigVerifier (check_schnorr_signatures / check_ecdsa_signatures)    crypto/txscript/src/lib.rs:574-643, batched
//   kgv::UtxoDiff (with_diff / diff_from / add_transaction)                 consensus/core/src/utxo/utxo_diff.rs:15-262
//   kgv::calc_hash_merkle_roots, kgv::check_block_bodies                    consensus/core/src/merkle.rs:5-7, body_validation_in_isolation.rs:95-131
//   kgv::BlockBodyProcessor (validate_body_in_isolation / validate_body_in_context / validate_bodies)  consensus/src/pipeline/body_processor/
//                                                                           body_validation_in_isolation.rs:13-131, body_validation_in_context.rs:20-80
// (* batched: one verdict per transaction.)  Verdicts are data (status codes of kgv.h); only transport failures throw.
// There is no CPU execution path behind any of this: without libkgv.so + a CUDA device, Context's constructor throws.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "kgv.h"

namespace kgv {

class Error : public std::runtime_error {
 public:
  Error(int code, const std::string& what) : std::runtime_error(what), code_(code) {}
  int code() const { return code_; }

 private:
  int code_;
};

// ---- data model (consensus/core/src/tx.rs) ----
using Hash = std::array<uint8_t, 32>;
using SubnetworkId = std::array<uint8_t, 20>;
inline SubnetworkId subnetwork_id_native() { return SubnetworkId{}; }
inline SubnetworkId subnetwork_id_coinbase() { SubnetworkId s{}; s[0] = 1; return s; }
struct ScriptPublicKey { uint16_t version = 0; std::vector<uint8_t> script; };
struct TransactionOutpoint { Hash transaction_id{}; uint32_t index = 0; };
struct TransactionInput { TransactionOutpoint previous_outpoint; std::vector<uint8_t> signature_script; uint64_t sequence = 0; uint8_t sig_op_count = 0; };
struct TransactionOutput { uint64_t value = 0; ScriptPublicKey script_public_key; };
struct UtxoEntry { uint64_t amount = 0; ScriptPublicKey script_public_key; uint64_t block_daa_score = 0; bool is_coinbase = false; };
struct Transaction {
  uint16_t version = 0;
  std::vector<TransactionInput> inputs;
  std::vector<TransactionOutput> outputs;
  uint64_t lock_time = 0;
  SubnetworkId subnetwork_id{};
  uint64_t gas = 0;
  std::vector<uint8_t> payload;
  uint64_t mass = 0;  // committed storage mass
};

// Flat SoA form of a list of (optionally populated) transactions: what crosses the ABI (INTEGRATION.md §2).
class TxBatch {
 public:
  // entries: nullptr, or for each transaction one optional entry per input (nullptr element = missing outpoint)
  void push(const Transaction& tx, const std::vector<const UtxoEntry*>* entries = nullptr) {
    kgv_tx t{};
    t.first_input = (uint32_t)inputs_.size();
    t.n_inputs = (uint32_t)tx.inputs.size();
    t.first_output = (uint32_t)outputs_.size();
    t.n_outputs = (uint32_t)tx.outputs.size();
    t.lock_time = tx.lock_time; t.gas = tx.gas; t.mass = tx.mass; t.version = tx.version;
    std::memcpy(t.subnetwork_id, tx.subnetwork_id.data(), 20);
    t.flags = tx.subnetwork_id == subnetwork_id_coinbase() ? 1 : 0;
    auto pl = put(tx.payload);
    t.payload_off = pl.first; t.payload_len = pl.second;
    for (size_t k = 0; k < tx.inputs.size(); k++) {
      const TransactionInput& in = tx.inputs[k];
      kgv_input r{};
      std::memcpy(r.prev_txid, in.previous_outpoint.transaction_id.data(), 32);
      r.prev_index = in.previous_outpoint.index;
      auto ss = put(in.signature_script);
      r.sigscript_off = ss.first; r.sigscript_len = ss.second;
      r.sig_op_count = in.sig_op_count; r.sequence = in.sequence;
      inputs_.push_back(r);
      kgv_utxo_entry e{};
      const UtxoEntry* ue = entries && k < entries->size() ? (*entries)[k] : nullptr;
      if (ue) {
        e.amount = ue->amount; e.block_daa_score = ue->block_daa_score; e.spk_version = ue->script_public_key.version; e.is_coinbase = ue->is_coinbase ? 1 : 0;
        auto sc = put(ue->script_public_key.script);
        e.script_off = sc.first; e.script_len = sc.second;
      } else {
        e.pad_[0] = 1;  // absent -> MissingTxOutpoints
      }
      entries_.push_back(e);
      populated_ = populated_ || entries != nullptr;
    }
    for (const TransactionOutput& o : tx.outputs) {
      kgv_output r{};
      r.value = o.value; r.spk_version = o.script_public_key.version;
      auto sc = put(o.script_public_key.script);
      r.script_off = sc.first; r.script_len = sc.second;
      outputs_.push_back(r);
    }
    txs_.push_back(t);
  }
  // adopt already-flat arrays (e.g. read from disk)
  void assign(std::vector<kgv_tx> txs, std::vector<kgv_input> inputs, std::vector<kgv_output> outputs, std::vector<kgv_utxo_entry> entries, std::vector<uint8_t> bytes) {
    txs_ = std::move(txs); inputs_ = std::move(inputs); outputs_ = std::move(outputs); entries_ = std::move(entries); bytes_ = std::move(bytes);
    populated_ = !entries_.empty();
  }
  size_t len() const { return txs_.size(); }
  size_t n_inputs() const { return inputs_.size(); }
  size_t n_outputs() const { return outputs_.size(); }
  kgv_tx_batch view(bool with_entries) const {
    kgv_tx_batch b{};
    b.txs = txs_.data(); b.n_txs = txs_.size();
    b.inputs = inputs_.data(); b.n_inputs = inputs_.size();
    b.outputs = outputs_.data(); b.n_outputs = outputs_.size();
    b.entries = (with_entries && populated_) ? entries_.data() : nullptr;
    b.bytes = bytes_.data(); b.n_bytes = bytes_.size();
    return b;
  }

 private:
  std::pair<uint32_t, uint32_t> put(const std::vector<uint8_t>& v) {
    uint32_t off = (uint32_t)bytes_.size();
    bytes_.insert(bytes_.end(), v.begin(), v.end());
    return {off, (uint32_t)v.size()};
  }
  std::vector<kgv_tx> txs_;
  std::vector<kgv_input> inputs_;
  std::vector<kgv_output> outputs_;
  std::vector<kgv_utxo_entry> entries_;
  std::vector<uint8_t> bytes_{0, 0, 0, 0, 0, 0, 0, 0};
  bool populated_ = false;
};

// ---- UTXO diff algebra (consensus/core/src/utxo/utxo_diff.rs:15-262, utxo_collection.rs): host bookkeeping, one diff per chain
// block; the GPU table consumes diffs through UtxoSet::write_diff.  Semantics pinned by the reference's rule table
// (tests/golden/utxo_diff_rules.json via tests/cpp/utxo_diff_test.cpp).
struct OutpointLess {
  bool operator()(const TransactionOutpoint& a, const TransactionOutpoint& b) const {
    return a.transaction_id != b.transaction_id ? a.transaction_id < b.transaction_id : a.index < b.index;
  }
};
inline bool operator==(const ScriptPublicKey& a, const ScriptPublicKey& b) { return a.version == b.version && a.script == b.script; }
inline bool operator==(const UtxoEntry& a, const UtxoEntry& b) {
  return a.amount == b.amount && a.script_public_key == b.script_public_key && a.block_daa_score == b.block_daa_score && a.is_coinbase == b.is_coinbase;
}
inline bool operator==(const TransactionOutpoint& a, const TransactionOutpoint& b) { return a.transaction_id == b.transaction_id && a.index == b.index; }
using UtxoCollection = std::map<TransactionOutpoint, UtxoEntry, OutpointLess>;

class UtxoAlgebraError : public std::runtime_error {
 public:
  enum Kind { DuplicateRemovePoint, DuplicateAddPoint, DoubleRemoveCall, DoubleAddCall, DiffIntersectionPoint, General };
  UtxoAlgebraError(Kind k, const char* name) : std::runtime_error(name), kind(k) {}
  Kind kind;
};

class UtxoDiff {
 public:
  UtxoCollection add, remove;
  bool operator==(const UtxoDiff& o) const { return add == o.add && remove == o.remove; }
  UtxoDiff to_reversed() const { UtxoDiff r; r.add = remove; r.remove = add; return r; }

  // self, then other, applied to one base set (utxo_diff.rs:76-116)
  UtxoDiff with_diff(const UtxoDiff& other) const { UtxoDiff c = *this; c.with_diff_in_place(other); return c; }
  void with_diff_in_place(const UtxoDiff& other) {
    for (const auto& kv : other.remove)
      if (remove.count(kv.first) && !has(add, kv.first, kv.second.block_daa_score)) throw UtxoAlgebraError(UtxoAlgebraError::DuplicateRemovePoint, "DuplicateRemovePoint");
    for (const auto& kv : other.add) {
      auto it = add.find(kv.first);
      if (it != add.end() && !has(other.remove, kv.first, it->second.block_daa_score)) throw UtxoAlgebraError(UtxoAlgebraError::DuplicateAddPoint, "DuplicateAddPoint");
    }
    std::vector<TransactionOutpoint> cancelled;
    for (const auto& kv : other.remove) {
      if (has(add, kv.first, kv.second.block_daa_score)) cancelled.push_back(kv.first);
      else remove[kv.first] = kv.second;
    }
    for (const auto& o : cancelled) add.erase(o);
    cancelled.clear();
    for (const auto& kv : other.add) {
      if (has(remove, kv.first, kv.second.block_daa_score)) cancelled.push_back(kv.first);
      else add[kv.first] = kv.second;
    }
    for (const auto& o : cancelled) remove.erase(o);
  }

  // the diff that turns self into other, both taken from one base set (utxo_diff.rs:118-225)
  UtxoDiff diff_from(const UtxoDiff& other) const {
    for (const auto& kv : remove) {
      auto it = other.add.find(kv.first);
      if (it == other.add.end()) continue;
      const uint64_t t = kv.second.block_daa_score, x = it->second.block_daa_score;
      if (!(x != t && (has(add, kv.first, x) || has(other.remove, kv.first, t)))) throw UtxoAlgebraError(UtxoAlgebraError::DiffIntersectionPoint, "DiffIntersectionPoint");
    }
    for (const auto& kv : add) {
      auto it = other.remove.find(kv.first);
      if (it == other.remove.end()) continue;
      const uint64_t t = kv.second.block_daa_score, x = it->second.block_daa_score;
      if (!(x != t && (has(remove, kv.first, x) || has(other.add, kv.first, t)))) throw UtxoAlgebraError(UtxoAlgebraError::DiffIntersectionPoint, "DiffIntersectionPoint");
    }
    for (const auto& kv : remove) {
      auto it = other.remove.find(kv.first);
      if (it != other.remove.end() && it->second.block_daa_score != kv.second.block_daa_score)
        throw UtxoAlgebraError(UtxoAlgebraError::DiffIntersectionPoint, "DiffIntersectionPoint");
    }
    UtxoDiff res;
    bool both_in_my_remove = false, both_in_other_remove = false;
    for (const auto& kv : add) {
      if (has(other.add, kv.first, kv.second.block_daa_score)) {
        both_in_my_remove = both_in_my_remove || remove.count(kv.first);
        both_in_other_remove = both_in_other_remove || other.remove.count(kv.first);
      } else {
        res.remove[kv.first] = kv.second;
      }
    }
    if (both_in_my_remove != both_in_other_remove) throw UtxoAlgebraError(UtxoAlgebraError::General, "General");
    for (const auto& kv : other.remove) if (!has(remove, kv.first, kv.second.block_daa_score)) res.remove[kv.first] = kv.second;
    for (const auto& kv : remove) if (!has(other.remove, kv.first, kv.second.block_daa_score)) res.add[kv.first] = kv.second;
    for (const auto& kv : other.add) if (!has(add, kv.first, kv.second.block_daa_score)) res.add[kv.first] = kv.second;
    return res;
  }

  // utxo_diff.rs:227-261; entries: the populated entry of every input
  void add_transaction(const Transaction& tx, const std::vector<UtxoEntry>& entries, const Hash& tx_id, uint64_t block_daa_score) {
    for (size_t i = 0; i < tx.inputs.size(); i++) {
      const TransactionOutpoint& o = tx.inputs[i].previous_outpoint;
      if (has(add, o, entries[i].block_daa_score)) add.erase(o);
      else if (!remove.count(o)) remove[o] = entries[i];
      else throw UtxoAlgebraError(UtxoAlgebraError::DoubleRemoveCall, "DoubleRemoveCall");
    }
    const bool cb = tx.subnetwork_id == subnetwork_id_coinbase();
    for (size_t k = 0; k < tx.outputs.size(); k++) {
      TransactionOutpoint o;
      o.transaction_id = tx_id; o.index = (uint32_t)k;
      UtxoEntry e;
      e.amount = tx.outputs[k].value; e.script_public_key = tx.outputs[k].script_public_key; e.block_daa_score = block_daa_score; e.is_coinbase = cb;
      if (has(remove, o, block_daa_score)) remove.erase(o);
      else if (!add.count(o)) add[o] = e;
      else throw UtxoAlgebraError(UtxoAlgebraError::DoubleAddCall, "DoubleAddCall");
    }
  }

 private:
  static bool has(const UtxoCollection& c, const TransactionOutpoint& o, uint64_t daa) {  // contains_with_daa_score
    auto it = c.find(o);
    return it != c.end() && it->second.block_daa_score == daa;
  }
};

// ---- context ----
class Context {
 public:
  explicit Context(int device = 0) {
    int rc = kgv_create(device, 0, &h_);
    if (rc != KGV_OK) throw Error(rc, "kgv_create failed: no usable CUDA device (this library has no CPU path)");
  }
  ~Context() { if (h_) kgv_destroy(h_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  kgv_ctx* get() const { return h_; }
  void check(int rc) const { if (rc != KGV_OK) throw Error(rc, std::string("libkgv: ") + kgv_last_error(h_)); }

 private:
  kgv_ctx* h_ = nullptr;
};

// ---- signatures: batch counterparts of check_schnorr_signature / check_ecdsa_signature ----
class SigVerifier {
 public:
  explicit SigVerifier(Context& c) : c_(c) {}
  // SoA byte arrays: pk 32*n (x-only) / 33*n (compressed), msg 32*n, sig 64*n.  Returns KGV_SIG_* per triple.
  std::vector<uint8_t> check_schnorr_signatures(const std::vector<uint8_t>& pk32, const std::vector<uint8_t>& msg32, const std::vector<uint8_t>& sig64) {
    size_t n = msg32.size() / 32;
    if (pk32.size() != 32 * n || sig64.size() != 64 * n) throw Error(KGV_ERR_ARG, "check_schnorr_signatures: array sizes disagree");
    std::vector<uint8_t> st(n);
    c_.check(kgv_schnorr_verify(c_.get(), pk32.data(), msg32.data(), sig64.data(), n, st.data()));
    return st;
  }
  std::vector<uint8_t> check_ecdsa_signatures(const std::vector<uint8_t>& pk33, const std::vector<uint8_t>& msg32, const std::vector<uint8_t>& sig64) {
    size_t n = msg32.size() / 32;
    if (pk33.size() != 33 * n || sig64.size() != 64 * n) throw Error(KGV_ERR_ARG, "check_ecdsa_signatures: array sizes disagree");
    std::vector<uint8_t> st(n);
    c_.check(kgv_ecdsa_verify(c_.get(), pk33.data(), msg32.data(), sig64.data(), n, st.data()));
    return st;
  }

 private:
  Context& c_;
};

// ---- MuHash ----
class MuHash {
 public:
  explicit MuHash(Context& c) : c_(&c) { numerator_[0] = 1; denominator_[0] = 1; }
  MuHash(Context& c, const std::array<uint8_t, 384>& num, const std::array<uint8_t, 384>& den) : c_(&c), numerator_(num), denominator_(den) {}
  MuHash& add_element(const std::vector<uint8_t>& data) { return update({data}, {}); }
  MuHash& remove_element(const std::vector<uint8_t>& data) { return update({}, {data}); }
  MuHash& update(const std::vector<std::vector<uint8_t>>& add, const std::vector<std::vector<uint8_t>>& remove) {
    std::vector<uint8_t> data, flags;
    std::vector<uint64_t> off{0};
    for (const auto& v : add) { data.insert(data.end(), v.begin(), v.end()); off.push_back(data.size()); flags.push_back(0); }
    for (const auto& v : remove) { data.insert(data.end(), v.begin(), v.end()); off.push_back(data.size()); flags.push_back(1); }
    if (flags.empty()) return *this;
    data.resize(data.size() + 8);
    MuHash part(*c_);
    c_->check(kgv_muhash_elements(c_->get(), data.data(), off.data(), flags.data(), flags.size(), part.numerator_.data(), part.denominator_.data()));
    return combine(part);
  }
  MuHash& combine(const MuHash& o) {
    c_->check(kgv_muhash_combine(c_->get(), numerator_.data(), denominator_.data(), o.numerator_.data(), o.denominator_.data()));
    return *this;
  }
  std::array<uint8_t, 384> serialize() { finalize(); return numerator_; }
  Hash finalize() {
    std::array<uint8_t, 384> ser{};
    Hash h{};
    c_->check(kgv_muhash_finalize(c_->get(), numerator_.data(), denominator_.data(), ser.data(), h.data()));
    numerator_ = ser;  // normalize(): numerator /= denominator, denominator = 1
    denominator_.fill(0); denominator_[0] = 1;
    return h;
  }
  const std::array<uint8_t, 384>& numerator() const { return numerator_; }
  const std::array<uint8_t, 384>& denominator() const { return denominator_; }

 private:
  Context* c_;
  std::array<uint8_t, 384> numerator_{}, denominator_{};
};

// ---- UTXO set on the GPU ----
class UtxoSet {
 public:
  UtxoSet(Context& c, uint64_t capacity_slots) : c_(c) { c_.check(kgv_utxo_create(c_.get(), capacity_slots, &h_)); }
  // UtxoViewComposition::compose (consensus/core/src/utxo/utxo_view.rs:22-35,45-50): a diff layer over `base`; this object then IS base ∘ diff:
  // reads fall through to the base, writes stay in the layer until commit() (write_diff_batch) or discard()
  UtxoSet(Context& c, UtxoSet& base, uint64_t capacity_slots) : c_(c) { c_.check(kgv_utxo_view_create(c_.get(), base.get(), capacity_slots, &h_)); view_ = true; }
  ~UtxoSet() { if (h_) kgv_utxo_destroy(c_.get(), h_); }
  void commit() { c_.check(kgv_utxo_view_commit(c_.get(), h_)); }
  void discard() { c_.check(kgv_utxo_view_discard(c_.get(), h_)); }
  bool is_view() const { return view_; }
  UtxoSet(const UtxoSet&) = delete;
  UtxoSet& operator=(const UtxoSet&) = delete;
  kgv_utxo_table* get() const { return h_; }
  // write_diff_batch: delete `removed`, then put `added`
  void write_diff(const std::vector<TransactionOutpoint>& removed, const std::vector<std::pair<TransactionOutpoint, UtxoEntry>>& added) {
    std::vector<uint8_t> rk(36 * removed.size()), ak(36 * added.size()), rs(removed.size() + 1), as(added.size() + 1), bytes(8);
    std::vector<kgv_utxo_entry> ae(added.size());
    for (size_t i = 0; i < removed.size(); i++) key36(rk.data() + 36 * i, removed[i]);
    for (size_t i = 0; i < added.size(); i++) {
      key36(ak.data() + 36 * i, added[i].first);
      const UtxoEntry& e = added[i].second;
      ae[i].amount = e.amount; ae[i].block_daa_score = e.block_daa_score; ae[i].spk_version = e.script_public_key.version; ae[i].is_coinbase = e.is_coinbase ? 1 : 0;
      ae[i].script_off = (uint32_t)bytes.size(); ae[i].script_len = (uint32_t)e.script_public_key.script.size();
      bytes.insert(bytes.end(), e.script_public_key.script.begin(), e.script_public_key.script.end());
    }
    c_.check(kgv_utxo_apply_diff(c_.get(), h_, removed.empty() ? nullptr : rk.data(), removed.size(), rs.data(), added.empty() ? nullptr : ak.data(),
                                 added.empty() ? nullptr : ae.data(), bytes.data(), bytes.size(), added.size(), as.data()));
  }
  // UtxoDiff::add_transaction for every accepted transaction of the batch
  void add_transactions(const TxBatch& b, const std::vector<uint8_t>& accept, uint64_t pov_daa_score) {
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_utxo_apply_accepted(c_.get(), h_, &v, accept.data(), pov_daa_score));
  }
  uint64_t count() { uint64_t n = 0; c_.check(kgv_utxo_count(c_.get(), h_, &n)); return n; }
  // maintenance: the table's state, an out-of-place rebuild (capacity 0 = same size), the opt-in growth policy (permille, 0 = off)
  kgv_utxo_table_stats stats() { kgv_utxo_table_stats s{}; c_.check(kgv_utxo_stats(c_.get(), h_, &s)); return s; }
  void rehash(uint64_t capacity_slots = 0) { c_.check(kgv_utxo_rehash(c_.get(), h_, capacity_slots)); }
  void set_max_load(uint32_t max_load_permille) { c_.check(kgv_utxo_set_max_load(c_.get(), h_, max_load_permille)); }
  // DbUtxoSetStore::iterator (consensus/src/model/stores/utxo_set.rs:114-129): every live entry, in the table's (arbitrary) order
  std::vector<std::pair<TransactionOutpoint, UtxoEntry>> iterator() {
    size_t n = 0, nb = 0;
    c_.check(kgv_utxo_export(c_.get(), h_, nullptr, nullptr, nullptr, 0, 0, &n, &nb));
    std::vector<uint8_t> keys(36 * n + 4), bytes(nb + 8);
    std::vector<kgv_utxo_entry> ent(n + 1);
    c_.check(kgv_utxo_export(c_.get(), h_, keys.data(), ent.data(), bytes.data(), n, nb, &n, &nb));
    std::vector<std::pair<TransactionOutpoint, UtxoEntry>> out(n);
    for (size_t i = 0; i < n; i++) {
      std::memcpy(out[i].first.transaction_id.data(), keys.data() + 36 * i, 32);
      out[i].first.index = 0;
      for (int b = 0; b < 4; b++) out[i].first.index |= (uint32_t)keys[36 * i + 32 + b] << (8 * b);
      UtxoEntry& e = out[i].second;
      e.amount = ent[i].amount; e.block_daa_score = ent[i].block_daa_score; e.is_coinbase = ent[i].is_coinbase != 0;
      e.script_public_key.version = ent[i].spk_version;
      e.script_public_key.script.assign(bytes.begin() + ent[i].script_off, bytes.begin() + ent[i].script_off + ent[i].script_len);
    }
    return out;
  }
  // Consensus::append_imported_pruning_point_utxos (consensus/src/consensus/mod.rs:1070-1083): the chunk goes into the set, MuHash::from_utxo of
  // its entries into `current_multiset` (whose denominator stays untouched)
  void append_imported_pruning_point_utxos(const std::vector<std::pair<TransactionOutpoint, UtxoEntry>>& chunk, MuHash& current_multiset) {
    if (chunk.empty()) return;
    std::vector<uint8_t> ak(36 * chunk.size()), bytes(8);
    std::vector<kgv_utxo_entry> ae(chunk.size());
    for (size_t i = 0; i < chunk.size(); i++) {
      key36(ak.data() + 36 * i, chunk[i].first);
      const UtxoEntry& e = chunk[i].second;
      std::memset(&ae[i], 0, sizeof ae[i]);
      ae[i].amount = e.amount; ae[i].block_daa_score = e.block_daa_score; ae[i].spk_version = e.script_public_key.version; ae[i].is_coinbase = e.is_coinbase ? 1 : 0;
      ae[i].script_off = (uint32_t)bytes.size(); ae[i].script_len = (uint32_t)e.script_public_key.script.size();
      bytes.insert(bytes.end(), e.script_public_key.script.begin(), e.script_public_key.script.end());
    }
    std::array<uint8_t, 384> num = current_multiset.numerator();
    c_.check(kgv_utxo_import_chunk(c_.get(), h_, ak.data(), ae.data(), bytes.data(), bytes.size(), chunk.size(), num.data()));
    current_multiset = MuHash(c_, num, current_multiset.denominator());
  }
  MuHash muhash() {
    std::array<uint8_t, 384> num{}, one{};
    one[0] = 1;
    c_.check(kgv_utxo_muhash(c_.get(), h_, num.data()));
    return MuHash(c_, num, one);
  }

 private:
  static void key36(uint8_t* k, const TransactionOutpoint& o) {
    std::memcpy(k, o.transaction_id.data(), 32);
    for (int i = 0; i < 4; i++) k[32 + i] = (uint8_t)(o.index >> (8 * i));
  }
  Context& c_;
  kgv_utxo_table* h_ = nullptr;
  bool view_ = false;
};

// ---- Cache<SigCacheKey, bool> (crypto/txscript/src/caches.rs:14-55): device-resident, attached to a context ----
class SigCache {
 public:
  SigCache(Context& c, uint64_t size = 10000) : c_(c) { c_.check(kgv_sigcache_create(c_.get(), size, &h_)); c_.check(kgv_set_sigcache(c_.get(), h_)); }
  ~SigCache() { if (h_) { kgv_set_sigcache(c_.get(), nullptr); kgv_sigcache_destroy(h_); } }
  SigCache(const SigCache&) = delete;
  SigCache& operator=(const SigCache&) = delete;
  void clear() { c_.check(kgv_sigcache_clear(c_.get(), h_)); }
  struct Counters { uint64_t get_counts, insert_counts, lookups, evictions; };  // caches.rs:57-93
  Counters counters() { Counters k{}; c_.check(kgv_sigcache_counters(c_.get(), h_, &k.get_counts, &k.insert_counts, &k.lookups, &k.evictions)); return k; }

 private:
  Context& c_;
  kgv_sigcache* h_ = nullptr;
};

// ---- prepared public keys kept across verify launches (kgv_keycache; no counterpart in the reference), shared by contexts of one device ----
// Each KeyCache attaches one context; the records live until the last one is destroyed, in any order.
class KeyCache {
 public:
  KeyCache(Context& c, uint64_t schnorr_keys, uint64_t ecdsa_keys) : c_(c) { c_.check(kgv_keycache_create(c_.get(), schnorr_keys, ecdsa_keys)); }
  // the cache of `holder`, attached to c as well (kgv_keycache_share): e.g. the block context's cache shared with the mempool's context
  KeyCache(Context& c, KeyCache& holder) : c_(c) { c_.check(kgv_keycache_share(c_.get(), holder.c_.get())); }
  ~KeyCache() { kgv_keycache_destroy(c_.get()); }
  KeyCache(const KeyCache&) = delete;
  KeyCache& operator=(const KeyCache&) = delete;
  void enable(bool on) { c_.check(kgv_set_keycache(c_.get(), on)); }
  void clear() { c_.check(kgv_keycache_clear(c_.get())); }
  struct Counters { uint64_t lookups, hits, inserts, evictions; };
  Counters counters(bool ecdsa) {
    Counters k{kgv_keycache_counter(c_.get(), ecdsa, KGV_KEYCACHE_LOOKUPS), kgv_keycache_counter(c_.get(), ecdsa, KGV_KEYCACHE_HITS),
               kgv_keycache_counter(c_.get(), ecdsa, KGV_KEYCACHE_INSERTS), kgv_keycache_counter(c_.get(), ecdsa, KGV_KEYCACHE_EVICTIONS)};
    if (k.lookups == UINT64_MAX || k.hits == UINT64_MAX || k.inserts == UINT64_MAX || k.evictions == UINT64_MAX) c_.check(KGV_ERR_CUDA);
    return k;
  }

 private:
  Context& c_;
};

// ---- transaction validation in UTXO context ----
struct Params {
  uint64_t coinbase_maturity = 100, storage_mass_parameter = 1000000000000ull, max_sompi = 2900000000000000000ull;  // consensus/core/src/config/params.rs, constants.rs
};
enum class TxValidationFlags : uint32_t { Full = KGV_FLAGS_FULL, SkipScriptChecks = KGV_FLAGS_SKIP_SCRIPT_CHECKS, SkipMassCheck = KGV_FLAGS_SKIP_MASS_CHECK };
// parameters of the isolation rules and the non-contextual masses: mainnet's (MAINNET_PARAMS, consensus/core/src/config/params.rs; ghostdag_k of 10 BPS)
struct TxRules : kgv_tx_rules {
  TxRules() : kgv_tx_rules{1000, 1000, 10000, 10000, 1, 10, 1000, 124, 150} {}
};
// the mempool Config fields of the standardness policy; the defaults are the reference's (mining/src/mempool/config.rs: 1 000 sompi/kg,
// TX_VERSION for both versions)
struct MempoolPolicy : kgv_mempool_policy {
  MempoolPolicy(uint64_t minimum_relay_transaction_fee = 1000, uint16_t minimum_standard_transaction_version = 0,
                uint16_t maximum_standard_transaction_version = 0)
      : kgv_mempool_policy{minimum_relay_transaction_fee, minimum_standard_transaction_version, maximum_standard_transaction_version, {0, 0, 0, 0}} {}
};

class TransactionValidator {
 public:
  TransactionValidator(Context& c, const Params& p) : c_(c) { p_.coinbase_maturity = p.coinbase_maturity; p_.storage_mass_parameter = p.storage_mass_parameter; p_.max_sompi = p.max_sompi; }
  // one verdict (status, script error, failing input, fee) per transaction of a populated batch
  std::vector<kgv_tx_result> validate_populated_transactions(const TxBatch& b, uint64_t pov_daa_score, TxValidationFlags flags = TxValidationFlags::Full, bool host_vm = true) {
    std::vector<kgv_tx_result> res(b.len());
    kgv_tx_batch v = b.view(true);
    c_.check(kgv_validate_populated(c_.get(), &v, pov_daa_score, (uint32_t)flags, &p_, res.data()));
    if (host_vm) check_scripts_host(v, res);
    return res;
  }
  std::vector<kgv_tx_result> validate_transactions_in_parallel(UtxoSet& utxo_view, const TxBatch& b, uint64_t pov_daa_score, TxValidationFlags flags = TxValidationFlags::Full) {
    std::vector<kgv_tx_result> res(b.len());
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_validate_txs(c_.get(), utxo_view.get(), &v, pov_daa_score, (uint32_t)flags, &p_, res.data()));
    return res;
  }
  // calculate_utxo_state / verify_expected_utxo_state for a WINDOW of blocks as one call (utxo_validation.rs:110-228): block b = transactions
  // [blocks[b].first_tx, +n_txs) of the batch (tx 0 = its coinbase); flags per block KGV_REPLAY_*.  Returns the per-transaction verdicts; `accept`
  // (optional) receives which transactions were folded into the set.
  std::vector<kgv_tx_result> replay_window(UtxoSet& utxo_view, const TxBatch& b, const std::vector<kgv_replay_block>& blocks, std::vector<uint8_t>* accept = nullptr,
                                           kgv_replay_stats* stats = nullptr) {
    std::vector<kgv_tx_result> res(b.len());
    if (accept) accept->assign(b.len(), 0);
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_replay_window(c_.get(), utxo_view.get(), &v, blocks.data(), blocks.size(), &p_, res.data(), accept ? accept->data() : nullptr, stats));
    return res;
  }
  // ctx.mergeset_diff (utxo_validation.rs:119,148) of every group of blocks of the window replay_window just processed: group g = blocks
  // [group_first[g], group_first[g+1]) (kgv_replay_diffs)
  std::vector<UtxoDiff> replay_diffs(const std::vector<uint32_t>& group_first) {
    if (group_first.size() < 2) return {};
    const size_t n_groups = group_first.size() - 1;
    std::vector<kgv_diff_range> ranges(n_groups);
    size_t nr = 0, na = 0, nb = 0;
    c_.check(kgv_replay_diffs(c_.get(), group_first.data(), n_groups, ranges.data(), nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, &nr, &na, &nb));
    std::vector<uint8_t> rk(36 * nr + 4), ak(36 * na + 4), bytes(nb + 8);
    std::vector<kgv_utxo_entry> re(nr + 1), ae(na + 1);
    c_.check(kgv_replay_diffs(c_.get(), group_first.data(), n_groups, ranges.data(), rk.data(), re.data(), ak.data(), ae.data(), bytes.data(), nr, na, nb, &nr, &na,
                              &nb));
    auto put = [&](UtxoCollection& c, const uint8_t* k, const kgv_utxo_entry& r) {
      TransactionOutpoint o;
      std::memcpy(o.transaction_id.data(), k, 32);
      for (int b = 0; b < 4; b++) o.index |= (uint32_t)k[32 + b] << (8 * b);
      UtxoEntry e;
      e.amount = r.amount; e.block_daa_score = r.block_daa_score; e.is_coinbase = r.is_coinbase != 0; e.script_public_key.version = r.spk_version;
      e.script_public_key.script.assign(bytes.begin() + r.script_off, bytes.begin() + r.script_off + r.script_len);
      c[o] = e;
    };
    std::vector<UtxoDiff> out(n_groups);
    for (size_t g = 0; g < n_groups; g++) {
      for (uint64_t i = ranges[g].first_remove; i < ranges[g].first_remove + ranges[g].n_remove; i++) put(out[g].remove, rk.data() + 36 * i, re[i]);
      for (uint64_t i = ranges[g].first_add; i < ranges[g].first_add + ranges[g].n_add; i++) put(out[g].add, ak.data() + 36 * i, ae[i]);
    }
    return out;
  }
  // verify_expected_utxo_state of every chain block of the window replay_window just processed (kgv_replay_verify_chain): group g = blocks
  // [group_first[g], group_first[g+1]), the selected parent first, the chain block's own body (KGV_REPLAY_VERIFY_ONLY) last.  One result per
  // group; block_fees (optional) receives every block's total_fees, multisets768 (optional) the running multiset after every group.
  std::vector<kgv_chain_result> verify_chain_blocks(const std::vector<uint32_t>& group_first, const std::vector<kgv_chain_header>& headers,
                                                    const std::vector<uint8_t>& merged_flags, const uint8_t init768[768], const kgv_tx_rules& rules,
                                                    const kgv_body_rules& body_rules, std::vector<uint64_t>* block_fees = nullptr,
                                                    std::vector<uint8_t>* multisets768 = nullptr) {
    const size_t n_groups = group_first.size() ? group_first.size() - 1 : 0;
    // the call reads one merged-flags byte and writes one fee per window block, and reads one header per group
    if (n_groups == 0 || merged_flags.size() != group_first.back() || headers.size() != n_groups)
      throw Error(KGV_ERR_ARG, "verify_chain_blocks: one header per group and one merged-flags byte per window block");
    std::vector<kgv_chain_result> res(n_groups);
    if (block_fees) block_fees->assign(merged_flags.size(), 0);
    if (multisets768) multisets768->assign(768 * n_groups, 0);
    c_.check(kgv_replay_verify_chain(c_.get(), group_first.data(), n_groups, headers.data(), merged_flags.data(), init768, &rules, &body_rules, res.data(),
                                     block_fees ? block_fees->data() : nullptr, multisets768 ? multisets768->data() : nullptr));
    return res;
  }
  // the NEXT window's range checks and upload under the current window's compute (kgv_batch_prefetch): call it with window i+1, then
  // replay_window with window i; `next` must stay alive and unchanged until it is replayed
  void prefetch(const TxBatch& next) {
    kgv_tx_batch v = next.view(false);
    c_.check(kgv_batch_prefetch(c_.get(), &v));
  }
  // validate_mempool_transactions_in_parallel (consensus/src/pipeline/virtual_processor/processor.rs:853-878): same kernels, but every
  // outcome is returned (Vec<TxResult<()>>); `fee` feeds the host-side feerate check (tx_validation_in_utxo_context.rs:63-73).
  // validate_mempool_transactions_in_utxo_context is the mempool's own rule set: caller entries first, mass computed, feerate threshold.
  std::vector<kgv_tx_result> validate_mempool_transactions_in_parallel(UtxoSet& virtual_utxo_view, const TxBatch& b, uint64_t virtual_daa_score,
                                                                     TxValidationFlags flags = TxValidationFlags::Full) {
    return validate_transactions_in_parallel(virtual_utxo_view, b, virtual_daa_score, flags);
  }
  // validate_mempool_transaction_in_utxo_context (utxo_validation.rs:341-397) for a batch (kgv_validate_mempool_txs).  The entries the batch
  // was pushed with win (an in-mempool parent's output: block_daa_score = u64::MAX); nullptr elements, or a batch pushed without entries, are
  // looked up in the view.  args: empty (no feerate thresholds) or one per transaction.  entries[i] = input i's final entry, or nothing.
  struct MempoolValidation {
    std::vector<kgv_tx_result> results;
    std::vector<uint64_t> storage_mass;
    std::vector<std::pair<bool, UtxoEntry>> entries;  // (found, entry) per input of the batch
  };
  MempoolValidation validate_mempool_transactions_in_utxo_context(UtxoSet& virtual_utxo_view, const TxBatch& b, uint64_t virtual_daa_score,
                                                                  const std::vector<kgv_mempool_tx_args>& args = {}) {
    if (!args.empty() && args.size() != b.len()) throw Error(KGV_ERR_ARG, "kgv: one kgv_mempool_tx_args per transaction");
    MempoolValidation out;
    out.results.resize(b.len());
    out.storage_mass.resize(b.len());
    std::vector<kgv_utxo_entry> ent(b.n_inputs() + 1);
    kgv_tx_batch v = b.view(true);
    size_t used = 0;
    std::vector<uint8_t> scripts(v.n_bytes + 128 * b.n_inputs() + 8);  // caller scripts come from the arena; a looked-up one usually fits 128 bytes
    auto call = [&] {
      return kgv_validate_mempool_txs(c_.get(), virtual_utxo_view.get(), &v, virtual_daa_score, &p_, args.empty() ? nullptr : args.data(), out.results.data(),
                                      out.storage_mass.data(), ent.data(), scripts.data(), scripts.size(), &used);
    };
    int rc = call();
    if (rc == KGV_ERR_NOMEM && used > scripts.size()) {  // reported before any signature is verified
      scripts.resize(used);
      rc = call();
    }
    c_.check(rc);
    out.entries.resize(b.n_inputs());
    for (size_t i = 0; i < b.n_inputs(); i++) {
      if (ent[i].pad_[0]) continue;
      UtxoEntry& e = out.entries[i].second;
      out.entries[i].first = true;
      e.amount = ent[i].amount; e.block_daa_score = ent[i].block_daa_score; e.is_coinbase = ent[i].is_coinbase != 0;
      e.script_public_key.version = ent[i].spk_version;
      e.script_public_key.script.assign(scripts.begin() + ent[i].script_off, scripts.begin() + ent[i].script_off + ent[i].script_len);
    }
    return out;
  }
  // validate_tx_in_isolation, then (finality) validate_tx_in_header_context_with_args(tx, ctx_daa_score, ctx_past_median_time), for every
  // transaction of the batch (kgv_validate_txs_in_isolation); masses receives calc_non_contextual_masses of each when given
  std::vector<kgv_tx_result> validate_tx_in_isolation(const TxBatch& b, const TxRules& rules = TxRules(), uint64_t ctx_daa_score = 0,
                                                      uint64_t ctx_past_median_time = 0, bool finality = true, std::vector<kgv_tx_masses>* masses = nullptr) {
    std::vector<kgv_tx_result> res(b.len());
    if (masses) masses->assign(b.len(), kgv_tx_masses{});
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_validate_txs_in_isolation(c_.get(), &v, &rules, ctx_daa_score, ctx_past_median_time, finality ? 0u : KGV_ISOLATION_SKIP_FINALITY, res.data(),
                                           masses ? masses->data() : nullptr));
    return res;
  }
  // validate_mempool_transactions_in_parallel (processor.rs:853-878; kgv_validate_mempool_txs_in_parallel): per transaction isolation,
  // finality, then validate_mempool_transactions_in_utxo_context.  Only args[i].feerate_threshold is read: the feerate divisor uses the
  // non-contextual masses computed in the call, returned in `masses`.
  struct FullMempoolValidation : MempoolValidation {
    std::vector<kgv_tx_masses> masses;
  };
  FullMempoolValidation validate_mempool_transactions_in_parallel_full(UtxoSet& virtual_utxo_view, const TxBatch& b, uint64_t virtual_daa_score,
                                                                       uint64_t virtual_past_median_time, const TxRules& rules = TxRules(),
                                                                       const std::vector<kgv_mempool_tx_args>& args = {}) {
    if (!args.empty() && args.size() != b.len()) throw Error(KGV_ERR_ARG, "kgv: one kgv_mempool_tx_args per transaction");
    FullMempoolValidation out;
    out.results.resize(b.len());
    out.storage_mass.resize(b.len());
    out.masses.resize(b.len());
    std::vector<kgv_utxo_entry> ent(b.n_inputs() + 1);
    kgv_tx_batch v = b.view(true);
    size_t used = 0;
    std::vector<uint8_t> scripts(v.n_bytes + 128 * b.n_inputs() + 8);
    auto call = [&] {
      return kgv_validate_mempool_txs_in_parallel(c_.get(), virtual_utxo_view.get(), &v, virtual_daa_score, virtual_past_median_time, &p_, &rules,
                                                  args.empty() ? nullptr : args.data(), out.results.data(), out.storage_mass.data(), out.masses.data(), ent.data(),
                                                  scripts.data(), scripts.size(), &used);
    };
    int rc = call();
    if (rc == KGV_ERR_NOMEM && used > scripts.size()) {
      scripts.resize(used);
      rc = call();
    }
    c_.check(rc);
    out.entries.resize(b.n_inputs());
    for (size_t i = 0; i < b.n_inputs(); i++) {
      if (ent[i].pad_[0]) continue;
      UtxoEntry& e = out.entries[i].second;
      out.entries[i].first = true;
      e.amount = ent[i].amount; e.block_daa_score = ent[i].block_daa_score; e.is_coinbase = ent[i].is_coinbase != 0;
      e.script_public_key.version = ent[i].spk_version;
      e.script_public_key.script.assign(scripts.begin() + ent[i].script_off, scripts.begin() + ent[i].script_off + ent[i].script_len);
    }
    return out;
  }

  // ---- the mempool's standardness policy (mining/src/mempool/check_transaction_standard.rs) ----
  // Each verdict comes with the number its NonStandardError carries beyond the index (`detail`, 0 for any other status).
  struct StandardResults {
    std::vector<kgv_tx_result> results;
    std::vector<uint64_t> detail;
  };
  // check_transaction_standard_in_isolation (kgv_check_txs_standard_in_isolation); masses: calculated_non_contextual_masses, one per tx
  StandardResults check_transaction_standard_in_isolation(const TxBatch& b, const std::vector<kgv_tx_masses>& masses,
                                                          const MempoolPolicy& policy = MempoolPolicy()) {
    if (masses.size() != b.len()) throw Error(KGV_ERR_ARG, "kgv: one kgv_tx_masses per transaction");
    StandardResults out{std::vector<kgv_tx_result>(b.len()), std::vector<uint64_t>(b.len())};
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_check_txs_standard_in_isolation(c_.get(), &v, &policy, masses.data(), out.results.data(), out.detail.data()));
    return out;
  }
  // check_transaction_standard_in_context (kgv_check_txs_standard_in_context) on a batch pushed with its entries: storage_mass is tx.mass(),
  // fee the calculated_fee, one each per tx
  StandardResults check_transaction_standard_in_context(const TxBatch& b, const std::vector<kgv_tx_masses>& masses, const std::vector<uint64_t>& storage_mass,
                                                        const std::vector<uint64_t>& fee, const MempoolPolicy& policy = MempoolPolicy()) {
    if (masses.size() != b.len() || storage_mass.size() != b.len() || fee.size() != b.len())
      throw Error(KGV_ERR_ARG, "kgv: one mass record, storage mass and fee per transaction");
    StandardResults out{std::vector<kgv_tx_result>(b.len()), std::vector<uint64_t>(b.len())};
    kgv_tx_batch v = b.view(true);
    c_.check(kgv_check_txs_standard_in_context(c_.get(), &v, &policy, masses.data(), storage_mass.data(), fee.data(), out.results.data(), out.detail.data()));
    return out;
  }
  // is_transaction_output_dust (kgv_outputs_dust) for every output of the batch, in batch order
  std::vector<bool> is_transaction_output_dust(const TxBatch& b, uint64_t minimum_relay_transaction_fee = 1000) {
    kgv_tx_batch v = b.view(false);
    std::vector<uint8_t> d(v.n_outputs + 1);
    c_.check(kgv_outputs_dust(c_.get(), &v, minimum_relay_transaction_fee, d.data()));
    return std::vector<bool>(d.begin(), d.begin() + v.n_outputs);
  }
  // validate_mempool_transactions_in_parallel_full with the standardness policy in the mempool's admission order
  // (kgv_validate_mempool_txs_with_policy); policy == nullptr is accept_non_standard = true
  struct PolicyMempoolValidation : FullMempoolValidation {
    std::vector<uint64_t> detail;
  };
  PolicyMempoolValidation validate_mempool_transactions_with_policy(UtxoSet& virtual_utxo_view, const TxBatch& b, uint64_t virtual_daa_score,
                                                                    uint64_t virtual_past_median_time, const MempoolPolicy* policy,
                                                                    const TxRules& rules = TxRules(), const std::vector<kgv_mempool_tx_args>& args = {}) {
    if (!args.empty() && args.size() != b.len()) throw Error(KGV_ERR_ARG, "kgv: one kgv_mempool_tx_args per transaction");
    PolicyMempoolValidation out;
    out.results.resize(b.len());
    out.storage_mass.resize(b.len());
    out.masses.resize(b.len());
    out.detail.resize(b.len());
    std::vector<kgv_utxo_entry> ent(b.n_inputs() + 1);
    kgv_tx_batch v = b.view(true);
    size_t used = 0;
    std::vector<uint8_t> scripts(v.n_bytes + 128 * b.n_inputs() + 8);
    auto call = [&] {
      return kgv_validate_mempool_txs_with_policy(c_.get(), virtual_utxo_view.get(), &v, virtual_daa_score, virtual_past_median_time, &p_, &rules,
                                                  args.empty() ? nullptr : args.data(), out.results.data(), out.storage_mass.data(), out.masses.data(), ent.data(),
                                                  scripts.data(), scripts.size(), &used, policy, out.detail.data());
    };
    int rc = call();
    if (rc == KGV_ERR_NOMEM && used > scripts.size()) {
      scripts.resize(used);
      rc = call();
    }
    c_.check(rc);
    out.entries.resize(b.n_inputs());
    for (size_t i = 0; i < b.n_inputs(); i++) {
      if (ent[i].pad_[0]) continue;
      UtxoEntry& e = out.entries[i].second;
      out.entries[i].first = true;
      e.amount = ent[i].amount; e.block_daa_score = ent[i].block_daa_score; e.is_coinbase = ent[i].is_coinbase != 0;
      e.script_public_key.version = ent[i].spk_version;
      e.script_public_key.script.assign(scripts.begin() + ent[i].script_off, scripts.begin() + ent[i].script_off + ent[i].script_len);
    }
    return out;
  }

  std::pair<std::vector<kgv_tx_result>, MuHash> validate_transactions_with_muhash_in_parallel(UtxoSet& utxo_view, const TxBatch& b, uint64_t pov_daa_score,
                                                                                            TxValidationFlags flags = TxValidationFlags::Full) {
    auto res = validate_transactions_in_parallel(utxo_view, b, pov_daa_score, flags);
    std::vector<uint8_t> accept(res.size());
    for (size_t i = 0; i < res.size(); i++) accept[i] = res[i].status == KGV_TX_OK;
    MuHash mh(c_);
    std::array<uint8_t, 384> num{}, den{};
    kgv_tx_batch v = b.view(false);
    c_.check(kgv_muhash_txs(c_.get(), utxo_view.get(), &v, accept.data(), pov_daa_score, num.data(), den.data()));
    return {std::move(res), MuHash(c_, num, den)};
  }

  // check_scripts with the full script engine on the GPU (kgv_check_scripts) for every tx of `res` reported KGV_TX_NEEDS_HOST_VM; the
  // results of the host engine, fee kept.  b must carry the populated entries.
  void check_scripts(const TxBatch& b, std::vector<kgv_tx_result>& res) {
    std::vector<uint32_t> idx;
    for (size_t i = 0; i < res.size(); i++) if (res[i].status == KGV_TX_NEEDS_HOST_VM) idx.push_back((uint32_t)i);
    if (idx.empty()) return;
    kgv_tx_batch v = b.view(true);
    std::vector<kgv_tx_result> out(idx.size());
    c_.check(kgv_check_scripts(c_.get(), &v, idx.data(), idx.size(), out.data()));
    for (size_t k = 0; k < idx.size(); k++) { uint64_t fee = res[idx[k]].fee; res[idx[k]] = out[k]; res[idx[k]].fee = fee; }
  }

 private:
  void check_scripts_host(const kgv_tx_batch& v, std::vector<kgv_tx_result>& res) {
    std::vector<uint32_t> idx;
    for (size_t i = 0; i < res.size(); i++) if (res[i].status == KGV_TX_NEEDS_HOST_VM) idx.push_back((uint32_t)i);
    if (idx.empty()) return;
    std::vector<kgv_tx_result> out(idx.size());
    c_.check(kgv_check_scripts_host(c_.get(), &v, idx.data(), idx.size(), out.data()));
    for (size_t k = 0; k < idx.size(); k++) { uint64_t fee = res[idx[k]].fee; res[idx[k]] = out[k]; res[idx[k]].fee = fee; }
  }
  Context& c_;
  kgv_params p_{};
};

// ---- block body helpers ----
inline std::vector<Hash> calc_hash_merkle_roots(Context& c, const TxBatch& b, const std::vector<uint32_t>& block_first_tx) {
  std::vector<Hash> roots(block_first_tx.size() - 1);
  kgv_tx_batch v = b.view(false);
  c.check(kgv_block_hash_merkle_roots(c.get(), &v, block_first_tx.data(), (uint32_t)roots.size(), roots.empty() ? nullptr : roots[0].data()));
  return roots;
}
inline std::vector<kgv_block_check> check_block_bodies(Context& c, const TxBatch& b, const std::vector<uint32_t>& block_first_tx) {
  std::vector<kgv_block_check> out(block_first_tx.size() - 1);
  kgv_tx_batch v = b.view(false);
  c.check(kgv_block_set_checks(c.get(), &v, block_first_tx.data(), (uint32_t)out.size(), out.data()));
  return out;
}

// ---- BlockBodyProcessor: every body rule for a window of blocks in one call (kgv_validate_block_bodies) ----
struct BodyRules : kgv_body_rules {
  BodyRules() : kgv_body_rules{500000, 204} {}  // MAINNET_PARAMS: max_block_mass, max_coinbase_payload_len
};
struct BlockBodyVerdicts {
  std::vector<kgv_body_result> results;  // the first failing rule of each block (KGV_BODY_*); a verdict is data, never an exception
  std::vector<kgv_block_masses> masses;  // the block's Mass; zeros unless the block is KGV_BODY_OK
  std::vector<Hash> hash_merkle_roots;   // calc_hash_merkle_root of each block, for RuleError::BadMerkleRoot(header's, calculated)
};
class BlockBodyProcessor {
 public:
  explicit BlockBodyProcessor(Context& c, const TxRules& rules = TxRules(), const BodyRules& body_rules = BodyRules()) : c_(c), rules_(rules), body_(body_rules) {}
  // block k = transactions [block_first_tx[k], block_first_tx[k + 1]) of b; headers[k]: what the rules read from its header and the stores.
  // check_parent_bodies_exist is a statuses-store query and stays with the caller.
  BlockBodyVerdicts validate_body_in_isolation(const TxBatch& b, const std::vector<uint32_t>& block_first_tx, const std::vector<kgv_block_header_ctx>& headers) {
    return validate_bodies(b, block_first_tx, headers, KGV_BODY_ISOLATION_ONLY);
  }
  // the whole order: a block failing an isolation rule reports that rule, as the reference never reaches the context stage for it
  BlockBodyVerdicts validate_body_in_context(const TxBatch& b, const std::vector<uint32_t>& block_first_tx, const std::vector<kgv_block_header_ctx>& headers) {
    return validate_bodies(b, block_first_tx, headers, 0);
  }
  BlockBodyVerdicts validate_bodies(const TxBatch& b, const std::vector<uint32_t>& block_first_tx, const std::vector<kgv_block_header_ctx>& headers, uint32_t flags) {
    if (block_first_tx.empty() || headers.size() != block_first_tx.size() - 1) throw Error(KGV_ERR_ARG, "BlockBodyProcessor: one header record per block");
    const size_t n = headers.size();
    BlockBodyVerdicts v{std::vector<kgv_body_result>(n), std::vector<kgv_block_masses>(n), std::vector<Hash>(n)};
    kgv_tx_batch view = b.view(false);
    c_.check(kgv_validate_block_bodies(c_.get(), &view, block_first_tx.data(), (uint32_t)n, headers.data(), &rules_, &body_, flags, v.results.data(), v.masses.data(),
                                       n ? v.hash_merkle_roots[0].data() : nullptr));
    return v;
  }

 private:
  Context& c_;
  TxRules rules_;
  BodyRules body_;
};

// ---- HeaderProcessor: header validation in isolation for a batch of headers (kgv_validate_headers_in_isolation) ----
struct Header {  // consensus/core/src/header.rs: the fields the header hash covers
  uint16_t version = 1;
  std::vector<std::vector<Hash>> parents_by_level;  // expanded: one entry per level
  Hash hash_merkle_root{}, accepted_id_merkle_root{}, utxo_commitment{}, pruning_point{};
  uint64_t timestamp = 0, nonce = 0, daa_score = 0, blue_score = 0;
  uint32_t bits = 0;
  std::array<uint8_t, 24> blue_work{};  // Uint192, big-endian
};
struct HeaderRules : kgv_header_rules {
  // constants::BLOCK_VERSION and MAINNET_PARAMS: timestamp_deviation_tolerance 132 s, max_block_parents 16, max_block_level 225
  HeaderRules() : kgv_header_rules{132, 0, 1, 16, 225, 0} {}
};
struct HeaderVerdicts {
  std::vector<kgv_header_result> results;  // the first failing rule (KGV_HEADER_*), the level and the PoW pass bit of every header
  std::vector<Hash> hashes;                // hashing::header::hash of every header
};
class HeaderProcessor {
 public:
  explicit HeaderProcessor(Context& c, const HeaderRules& rules = HeaderRules()) : c_(c), rules_(rules) {}
  // validate_header_in_isolation (pre_ghostdag_validation.rs:17-24) of every header; the caller maps the statuses to RuleError and keeps
  // the level for parents_by_level and its stores.  now_ms stands for unix_now().
  HeaderVerdicts validate_headers_in_isolation(const std::vector<Header>& headers, uint64_t now_ms) {
    Packed p(headers);
    kgv_header_rules r = rules_;
    r.now_ms = now_ms;
    HeaderVerdicts v{std::vector<kgv_header_result>(headers.size()), std::vector<Hash>(headers.size())};
    c_.check(kgv_validate_headers_in_isolation(c_.get(), p.recs.data(), p.recs.size(), p.parents.empty() ? nullptr : p.parents[0].data(), p.parents.size(),
                                               p.lens.empty() ? nullptr : p.lens.data(), p.lens.size(), &r, v.results.data(),
                                               headers.empty() ? nullptr : v.hashes[0].data(), nullptr));
    return v;
  }
  // hashing::header::hash of every header (kgv_hash_headers)
  std::vector<Hash> hash_headers(const std::vector<Header>& headers) {
    Packed p(headers);
    std::vector<Hash> out(headers.size());
    c_.check(kgv_hash_headers(c_.get(), p.recs.data(), p.recs.size(), p.parents.empty() ? nullptr : p.parents[0].data(), p.parents.size(),
                              p.lens.empty() ? nullptr : p.lens.data(), p.lens.size(), headers.empty() ? nullptr : out[0].data(), nullptr));
    return out;
  }

 private:
  struct Packed {  // the C records and the parents arena
    std::vector<kgv_header> recs;
    std::vector<Hash> parents;
    std::vector<uint32_t> lens;
    explicit Packed(const std::vector<Header>& hs) : recs(hs.size()) {
      for (size_t k = 0; k < hs.size(); k++) {
        const Header& h = hs[k];
        kgv_header& r = recs[k];
        std::memset(&r, 0, sizeof r);
        std::memcpy(r.hash_merkle_root, h.hash_merkle_root.data(), 32);
        std::memcpy(r.accepted_id_merkle_root, h.accepted_id_merkle_root.data(), 32);
        std::memcpy(r.utxo_commitment, h.utxo_commitment.data(), 32);
        std::memcpy(r.pruning_point, h.pruning_point.data(), 32);
        std::memcpy(r.blue_work, h.blue_work.data(), 24);
        r.timestamp = h.timestamp; r.nonce = h.nonce; r.daa_score = h.daa_score; r.blue_score = h.blue_score; r.bits = h.bits; r.version = h.version;
        r.parents_off = parents.size();
        r.levels_off = (uint32_t)lens.size();
        r.n_levels = (uint32_t)h.parents_by_level.size();
        for (const auto& lvl : h.parents_by_level) {
          lens.push_back((uint32_t)lvl.size());
          parents.insert(parents.end(), lvl.begin(), lvl.end());
        }
      }
    }
  };
  Context& c_;
  HeaderRules rules_;
};

}  // namespace kgv
