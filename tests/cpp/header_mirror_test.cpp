// Validates dumped headers through the C++ host mirror (include/kgv.hpp, kgv::HeaderProcessor) and prints every verdict, for
// tests/test_gpu_cpp_headers.py to compare with the Python binding.  Needs a GPU to run.
//   header_mirror_test <dir> <now_ms> <max_block_parents> <max_block_level> <timestamp_deviation_tolerance>
// <dir> holds headers.bin (kgv_header records), lens.bin (u32 level sizes) and parents.bin (32-byte hashes), the arena of include/kgv.h.
// Output, per header: "<status> <level> <pow_passed> <a> <b> <hash hex>", then one line with the hashes of hash_headers, space-separated.
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
  if (argc < 6) { std::fprintf(stderr, "usage: %s <dir> <now_ms> <max_block_parents> <max_block_level> <tolerance>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  try {
    const auto recs = slurp<kgv_header>(dir + "headers.bin");
    const auto lens = slurp<uint32_t>(dir + "lens.bin");
    const auto parents = slurp<kgv::Hash>(dir + "parents.bin");
    // back to the mirror's data model: the processor packs its own arena
    std::vector<kgv::Header> hs(recs.size());
    for (size_t k = 0; k < recs.size(); k++) {
      const kgv_header& r = recs[k];
      kgv::Header& h = hs[k];
      h.version = r.version; h.timestamp = r.timestamp; h.nonce = r.nonce; h.daa_score = r.daa_score; h.blue_score = r.blue_score; h.bits = r.bits;
      std::memcpy(h.hash_merkle_root.data(), r.hash_merkle_root, 32);
      std::memcpy(h.accepted_id_merkle_root.data(), r.accepted_id_merkle_root, 32);
      std::memcpy(h.utxo_commitment.data(), r.utxo_commitment, 32);
      std::memcpy(h.pruning_point.data(), r.pruning_point, 32);
      std::memcpy(h.blue_work.data(), r.blue_work, 24);
      size_t p = r.parents_off;
      for (uint32_t l = 0; l < r.n_levels; l++) {
        const uint32_t n = lens[r.levels_off + l];
        h.parents_by_level.emplace_back(parents.begin() + p, parents.begin() + p + n);
        p += n;
      }
    }
    kgv::Context ctx(0);
    kgv::HeaderRules rules;
    rules.max_block_parents = (uint32_t)std::stoul(argv[3]);
    rules.max_block_level = (uint32_t)std::stoul(argv[4]);
    rules.timestamp_deviation_tolerance = std::stoull(argv[5]);
    kgv::HeaderProcessor hp(ctx, rules);
    const auto v = hp.validate_headers_in_isolation(hs, std::stoull(argv[2]));
    for (size_t k = 0; k < hs.size(); k++) {
      const kgv_header_result& r = v.results[k];
      std::cout << r.status << " " << (int)r.level << " " << (int)r.pow_passed << " " << r.a << " " << r.b << " " << hex(v.hashes[k].data(), 32) << "\n";
    }
    const auto hh = hp.hash_headers(hs);
    for (size_t k = 0; k < hh.size(); k++) std::cout << (k ? " " : "") << hex(hh[k].data(), 32);
    std::cout << "\n";
  } catch (const std::exception& e) {
    std::cerr << "error: " << e.what() << "\n";
    return 1;
  }
  return 0;
}
