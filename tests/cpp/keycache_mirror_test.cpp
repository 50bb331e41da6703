// Exercises kgv::KeyCache of the C++ host mirror (include/kgv.hpp) on triples dumped by tests/test_gpu_cpp_keycache.py: the same Schnorr
// and ECDSA batches verified twice (cold, then warm) with the cache attached, then once after clear().  Prints every verdict line and the
// counters of both kinds as plain text for the Python side to compare.
//   keycache_mirror_test <dir>      (<dir>: s_pk.bin s_msg.bin s_sig.bin e_pk.bin e_msg.bin e_sig.bin)
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>

#include "../../include/kgv.hpp"

static std::vector<uint8_t> slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::runtime_error("cannot open " + path);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
static void line(const char* tag, const std::vector<uint8_t>& st) {
  printf("%s", tag);
  for (uint8_t s : st) printf(" %d", s);
  printf("\n");
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string d = argv[1];
  try {
    kgv::Context ctx(0);
    kgv::SigVerifier v(ctx);
    const auto spk = slurp(d + "/s_pk.bin"), smsg = slurp(d + "/s_msg.bin"), ssig = slurp(d + "/s_sig.bin");
    const auto epk = slurp(d + "/e_pk.bin"), emsg = slurp(d + "/e_msg.bin"), esig = slurp(d + "/e_sig.bin");
    {
      kgv::KeyCache kc(ctx, 1024, 1024);
      for (const char* pass : {"cold", "warm"}) {
        line((std::string("schnorr_") + pass).c_str(), v.check_schnorr_signatures(spk, smsg, ssig));
        line((std::string("ecdsa_") + pass).c_str(), v.check_ecdsa_signatures(epk, emsg, esig));
      }
      for (int e = 0; e < 2; e++) {
        const auto c = kc.counters(e);
        printf("counters %d %llu %llu %llu %llu\n", e, (unsigned long long)c.lookups, (unsigned long long)c.hits, (unsigned long long)c.inserts,
               (unsigned long long)c.evictions);
      }
      kc.clear();
      line("schnorr_cleared", v.check_schnorr_signatures(spk, smsg, ssig));
      const auto c = kc.counters(false);
      printf("cleared %llu %llu\n", (unsigned long long)c.lookups, (unsigned long long)c.hits);
    }  // destroyed: detached from the context
    line("schnorr_detached", v.check_schnorr_signatures(spk, smsg, ssig));
  } catch (const std::exception& e) {
    printf("error %s\n", e.what());
    return 1;
  }
  return 0;
}
