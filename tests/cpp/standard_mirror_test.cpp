// Exercises the standardness methods of the C++ host mirror (include/kgv.hpp: MempoolPolicy, TransactionValidator::
// check_transaction_standard_in_isolation / _in_context, is_transaction_output_dust, validate_mempool_transactions_with_policy) on batches
// dumped by tests/test_gpu_cpp_standard.py, and prints the outcome as plain text for the Python side to compare.  Built by that test (g++,
// links libkgv.so); needs a GPU to run.
//   standard_mirror_test <dir> <relay fee>
// <dir> holds, per section s in {iso, ctx, dust, pol}: s_txs.bin s_inputs.bin s_outputs.bin s_entries.bin s_arena.bin (flat records of
// include/kgv.h), and iso_masses.bin, ctx_masses.bin ctx_smass.bin ctx_fee.bin.  Output lines:
//   iso <k> <status> <fail_input> <detail>            ctx <k> <status> <fail_input> <detail> <fee>
//   dust <o> <0|1>                                    pol <k> <status> <fail_input> <detail> <storage_mass> <compute_mass> <transient_mass>
//   threw                                             (the relay-fee overflow of the context check raised kgv::Error)
#include <cstdio>
#include <fstream>
#include <iostream>

#include "../../include/kgv.hpp"

template <class T>
static std::vector<T> slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::runtime_error("cannot open " + path);
  std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  std::vector<T> v(raw.size() / sizeof(T));
  std::memcpy(v.data(), raw.data(), v.size() * sizeof(T));
  return v;
}

static kgv::TxBatch batch(const std::string& p) {
  kgv::TxBatch b;
  b.assign(slurp<kgv_tx>(p + "txs.bin"), slurp<kgv_input>(p + "inputs.bin"), slurp<kgv_output>(p + "outputs.bin"), slurp<kgv_utxo_entry>(p + "entries.bin"),
           slurp<uint8_t>(p + "arena.bin"));
  return b;
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s <dir> <relay fee>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  const kgv::MempoolPolicy policy(std::stoull(argv[2]));
  try {
    kgv::Context ctx(0);
    kgv::TransactionValidator tv(ctx, kgv::Params());
    auto iso = tv.check_transaction_standard_in_isolation(batch(dir + "iso_"), slurp<kgv_tx_masses>(dir + "iso_masses.bin"), policy);
    for (size_t k = 0; k < iso.results.size(); k++)
      std::cout << "iso " << k << " " << (int)iso.results[k].status << " " << iso.results[k].fail_input << " " << iso.detail[k] << "\n";
    const auto cm = slurp<kgv_tx_masses>(dir + "ctx_masses.bin");
    const auto cs = slurp<uint64_t>(dir + "ctx_smass.bin");
    const auto cf = slurp<uint64_t>(dir + "ctx_fee.bin");
    const kgv::TxBatch cb = batch(dir + "ctx_");
    auto cx = tv.check_transaction_standard_in_context(cb, cm, cs, cf, policy);
    for (size_t k = 0; k < cx.results.size(); k++)
      std::cout << "ctx " << k << " " << (int)cx.results[k].status << " " << cx.results[k].fail_input << " " << cx.detail[k] << " " << cx.results[k].fee << "\n";
    auto dust = tv.is_transaction_output_dust(batch(dir + "dust_"), policy.minimum_relay_transaction_fee);
    for (size_t o = 0; o < dust.size(); o++) std::cout << "dust " << o << " " << (dust[o] ? 1 : 0) << "\n";
    kgv::UtxoSet us(ctx, 1 << 10);  // empty: the batch supplies every entry
    auto pol = tv.validate_mempool_transactions_with_policy(us, batch(dir + "pol_"), 1000, 0, &policy);
    for (size_t k = 0; k < pol.results.size(); k++)
      std::cout << "pol " << k << " " << (int)pol.results[k].status << " " << pol.results[k].fail_input << " " << pol.detail[k] << " " << pol.storage_mass[k] << " "
                << pol.masses[k].compute_mass << " " << pol.masses[k].transient_mass << "\n";
    try {
      std::vector<kgv_tx_masses> big(cm.size(), kgv_tx_masses{2, 0});
      tv.check_transaction_standard_in_context(cb, big, cs, cf, kgv::MempoolPolicy(~0ull));
    } catch (const kgv::Error&) {
      std::cout << "threw\n";
    }
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
