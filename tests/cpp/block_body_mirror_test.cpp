// Exercises kgv::BlockBodyProcessor of the C++ host mirror (include/kgv.hpp) on data dumped by tests/test_gpu_cpp_block_bodies.py and prints
// the outcome as plain text for the Python side to compare with the oracle.  Built by that test (g++, links libkgv.so); needs a GPU to run.
//   block_body_mirror_test <dir> <max_block_mass>
// <dir> holds txs.bin inputs.bin outputs.bin arena.bin (flat records of include/kgv.h), blocks.bin (u32 offsets) and headers.bin
// (kgv_block_header_ctx records).  Output, per block: "iso <status> <index> <tx_status> <fail_input> <a> <b> <compute> <transient> <storage>"
// from validate_body_in_isolation, then the same with "ctx" and the root in hex from validate_body_in_context.
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

static void print(const char* tag, const kgv::BlockBodyVerdicts& v, bool roots) {
  for (size_t k = 0; k < v.results.size(); k++) {
    const kgv_body_result& r = v.results[k];
    std::cout << tag << " " << r.status << " " << r.index << " " << r.tx_status << " " << r.fail_input << " " << r.a << " " << r.b << " " << v.masses[k].compute_mass << " "
              << v.masses[k].transient_mass << " " << v.masses[k].storage_mass;
    if (roots) {
      std::cout << " ";
      for (uint8_t b : v.hash_merkle_roots[k]) std::printf("%02x", b);
      std::fflush(stdout);
    }
    std::cout << std::endl;
  }
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s <dir> <max_block_mass>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  try {
    kgv::Context ctx(0);
    kgv::BodyRules body;
    body.max_block_mass = std::stoull(argv[2]);
    kgv::BlockBodyProcessor bp(ctx, kgv::TxRules(), body);
    kgv::TxBatch b;
    b.assign(slurp<kgv_tx>(dir + "txs.bin"), slurp<kgv_input>(dir + "inputs.bin"), slurp<kgv_output>(dir + "outputs.bin"), {}, slurp<uint8_t>(dir + "arena.bin"));
    const auto first = slurp<uint32_t>(dir + "blocks.bin");
    const auto headers = slurp<kgv_block_header_ctx>(dir + "headers.bin");
    print("iso", bp.validate_body_in_isolation(b, first, headers), false);
    print("ctx", bp.validate_body_in_context(b, first, headers), true);
    try {  // a transport failure throws: one header short
      bp.validate_body_in_context(b, first, std::vector<kgv_block_header_ctx>(headers.begin(), headers.end() - 1));
      std::cout << "nothrow" << std::endl;
    } catch (const kgv::Error&) {
      std::cout << "threw" << std::endl;
    }
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
