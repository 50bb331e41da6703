// Replays one window through the C++ host mirror (include/kgv.hpp) and prints the UtxoDiff of every group of blocks
// (TransactionValidator::replay_diffs), for tests/test_gpu_replay_diffs.py to compare with the Python binding.  Needs a GPU to run.
//   replay_diffs_test <dir> <coinbase_maturity> <storage_mass_parameter>
// <dir> holds txs.bin inputs.bin outputs.bin arena.bin (flat records of include/kgv.h), blocks.bin (kgv_replay_block records) and
// groups.bin (u32 group offsets).  Output, per group, its additions then its removals in outpoint order:
//   "<group> add|rem <txid hex> <index> <amount> <block_daa_score> <is_coinbase> <spk_version> <script hex>"
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
    kgv::UtxoSet set(ctx, 1 << 12);
    kgv::TransactionValidator tv(ctx, prm);
    tv.replay_window(set, b, blocks);
    const std::vector<kgv::UtxoDiff> diffs = tv.replay_diffs(groups);
    for (size_t g = 0; g < diffs.size(); g++) {
      for (const char* side : {"add", "rem"}) {
        const kgv::UtxoCollection& c = side[0] == 'a' ? diffs[g].add : diffs[g].remove;
        for (const auto& kv : c) {
          const kgv::UtxoEntry& e = kv.second;
          std::cout << g << " " << side << " " << hex(kv.first.transaction_id.data(), 32) << " " << kv.first.index << " " << e.amount << " " << e.block_daa_score
                    << " " << (e.is_coinbase ? 1 : 0) << " " << e.script_public_key.version << " "
                    << hex(e.script_public_key.script.data(), e.script_public_key.script.size()) << "\n";
        }
      }
    }
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
