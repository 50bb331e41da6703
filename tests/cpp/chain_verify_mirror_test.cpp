// Replays one window through the C++ host mirror (include/kgv.hpp) and prints every chain block's verdict
// (TransactionValidator::verify_chain_blocks), for tests/test_gpu_chain_verify.py to compare with the Python binding.  Needs a GPU to run.
//   chain_verify_mirror_test <dir> <coinbase_maturity> <storage_mass_parameter>
// <dir> holds txs.bin inputs.bin outputs.bin arena.bin (flat records of include/kgv.h), blocks.bin (kgv_replay_block records), groups.bin
// (u32 group offsets), headers.bin (kgv_chain_header records), merged.bin (one KGV_MERGED_* byte per block) and init.bin (768 bytes).
// Output, per group: "<status> <n_invalid_txs> <n_txs> <commitment hex> <accepted-id root hex> <coinbase hash hex>", then one line of the
// block fees and one of the hex of the last running multiset.
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
static std::string hex(const uint8_t* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) { s.push_back(d[p[i] >> 4]); s.push_back(d[p[i] & 15]); }
  return s;
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: %s <dir> <coinbase_maturity> <storage_mass_parameter>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  try {
    kgv::Context ctx(0);
    kgv::Params prm;
    prm.coinbase_maturity = std::stoull(argv[2]);
    prm.storage_mass_parameter = std::stoull(argv[3]);
    kgv::TxBatch b;
    b.assign(slurp<kgv_tx>(dir + "txs.bin"), slurp<kgv_input>(dir + "inputs.bin"), slurp<kgv_output>(dir + "outputs.bin"), {}, slurp<uint8_t>(dir + "arena.bin"));
    const auto blocks = slurp<kgv_replay_block>(dir + "blocks.bin");
    const auto groups = slurp<uint32_t>(dir + "groups.bin");
    const auto headers = slurp<kgv_chain_header>(dir + "headers.bin");
    const auto merged = slurp<uint8_t>(dir + "merged.bin");
    const auto init = slurp<uint8_t>(dir + "init.bin");
    kgv::UtxoSet set(ctx, 1 << 16);
    kgv::TransactionValidator tv(ctx, prm);
    tv.replay_window(set, b, blocks);
    std::vector<uint64_t> fees;
    std::vector<uint8_t> ms;
    const auto res = tv.verify_chain_blocks(groups, headers, merged, init.data(), kgv::TxRules(), kgv::BodyRules(), &fees, &ms);
    for (const kgv_chain_result& r : res)
      std::cout << r.status << " " << r.n_invalid_txs << " " << r.n_txs << " " << hex(r.utxo_commitment, 32) << " " << hex(r.accepted_id_merkle_root, 32) << " "
                << hex(r.coinbase_hash, 32) << "\n";
    for (size_t i = 0; i < fees.size(); i++) std::cout << (i ? " " : "") << fees[i];
    std::cout << "\n" << hex(ms.data() + ms.size() - 768, 768) << "\n";
    // a merged_flags array that does not cover the window is refused by the mirror
    bool threw = false;
    try {
      tv.verify_chain_blocks(groups, headers, std::vector<uint8_t>(merged.begin(), merged.end() - 1), init.data(), kgv::TxRules(), kgv::BodyRules());
    } catch (const std::exception&) {
      threw = true;
    }
    std::cout << (threw ? "threw" : "accepted") << "\n";
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
