// Exercises TransactionValidator::check_scripts of the C++ host mirror (include/kgv.hpp): a populated batch dumped by
// tests/test_gpu_script_engine.py is validated with kgv_validate_populated (no host engine), and the transactions it leaves as
// KGV_TX_NEEDS_HOST_VM are decided by the device script engine.  Built by __graft_entry__.build() (g++, links libkgv.so); needs a GPU.
//   script_engine_mirror_test <dir> <pov_daa_score>
// <dir> holds txs.bin inputs.bin outputs.bin entries.bin arena.bin (flat records of include/kgv.h).  Output: one line per transaction
// "tx <status_before> <status> <script_err> <fail_input> <fee>".
#include <cstdio>
#include <cstring>
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

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s <dir> <pov_daa_score>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  try {
    kgv::Context ctx(0);
    kgv::Params p;
    p.coinbase_maturity = 0;
    p.storage_mass_parameter = 0;
    kgv::TransactionValidator tv(ctx, p);
    kgv::TxBatch b;
    b.assign(slurp<kgv_tx>(dir + "txs.bin"), slurp<kgv_input>(dir + "inputs.bin"), slurp<kgv_output>(dir + "outputs.bin"),
             slurp<kgv_utxo_entry>(dir + "entries.bin"), slurp<uint8_t>(dir + "arena.bin"));
    auto res = tv.validate_populated_transactions(b, std::stoull(argv[2]), kgv::TxValidationFlags::SkipMassCheck, false);
    const std::vector<kgv_tx_result> before = res;
    tv.check_scripts(b, res);
    for (size_t i = 0; i < res.size(); i++)
      std::cout << "tx " << (int)before[i].status << " " << (int)res[i].status << " " << (int)res[i].script_err << " " << res[i].fail_input << " " << res[i].fee << "\n";
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
