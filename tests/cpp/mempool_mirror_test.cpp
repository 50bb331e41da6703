// Exercises TransactionValidator::validate_mempool_transactions_in_utxo_context of the C++ host mirror (include/kgv.hpp) on data dumped by
// tests/test_gpu_mempool.py and prints the outcome as plain text for the Python side to compare with the oracle.  Built by that test
// (g++, links libkgv.so); needs a GPU to run.
//   mempool_mirror_test <dir> <virtual_daa_score> <storage_mass_parameter>
// <dir> holds txs.bin inputs.bin outputs.bin entries.bin arena.bin (flat records of include/kgv.h; an entry with pad_[0] != 0 is looked up),
// args.bin (one kgv_mempool_tx_args per transaction, or empty: no thresholds), fund_keys.bin fund_entries.bin fund_arena.bin (the virtual
// UTXO set).  Output: one line per transaction "tx <status> <script_err> <fail_input> <fee> <storage_mass>", then one per input
// "in <found> <amount> <block_daa_score> <spk_version> <is_coinbase> <script hex>".
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
static std::string hex(const std::vector<uint8_t>& v) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (uint8_t b : v) { s.push_back(d[b >> 4]); s.push_back(d[b & 15]); }
  return s.empty() ? "-" : s;
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: %s <dir> <virtual_daa_score> <storage_mass_parameter>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  try {
    kgv::Context ctx(0);
    kgv::Params p;
    p.coinbase_maturity = 4;
    p.storage_mass_parameter = std::stoull(argv[3]);
    kgv::TransactionValidator tv(ctx, p);
    kgv::UtxoSet us(ctx, 1 << 14);
    {
      auto keys = slurp<uint8_t>(dir + "fund_keys.bin");
      auto ents = slurp<kgv_utxo_entry>(dir + "fund_entries.bin");
      auto arena = slurp<uint8_t>(dir + "fund_arena.bin");
      std::vector<std::pair<kgv::TransactionOutpoint, kgv::UtxoEntry>> added;
      for (size_t i = 0; i < ents.size(); i++) {
        kgv::TransactionOutpoint o;
        std::memcpy(o.transaction_id.data(), &keys[36 * i], 32);
        for (int b = 0; b < 4; b++) o.index |= (uint32_t)keys[36 * i + 32 + b] << (8 * b);
        kgv::UtxoEntry e;
        e.amount = ents[i].amount; e.block_daa_score = ents[i].block_daa_score; e.is_coinbase = ents[i].is_coinbase != 0;
        e.script_public_key.version = ents[i].spk_version;
        e.script_public_key.script.assign(arena.begin() + ents[i].script_off, arena.begin() + ents[i].script_off + ents[i].script_len);
        added.emplace_back(o, e);
      }
      us.write_diff({}, added);
    }
    kgv::TxBatch b;
    b.assign(slurp<kgv_tx>(dir + "txs.bin"), slurp<kgv_input>(dir + "inputs.bin"), slurp<kgv_output>(dir + "outputs.bin"),
             slurp<kgv_utxo_entry>(dir + "entries.bin"), slurp<uint8_t>(dir + "arena.bin"));
    auto args = slurp<kgv_mempool_tx_args>(dir + "args.bin");
    auto r = tv.validate_mempool_transactions_in_utxo_context(us, b, std::stoull(argv[2]), args);
    for (size_t i = 0; i < r.results.size(); i++)
      std::cout << "tx " << (int)r.results[i].status << " " << (int)r.results[i].script_err << " " << r.results[i].fail_input << " " << r.results[i].fee << " "
                << r.storage_mass[i] << "\n";
    for (auto& e : r.entries)
      std::cout << "in " << (e.first ? 1 : 0) << " " << e.second.amount << " " << e.second.block_daa_score << " " << e.second.script_public_key.version << " "
                << (e.second.is_coinbase ? 1 : 0) << " " << hex(e.second.script_public_key.script) << "\n";
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
