// One kgv::KeyCache shared by two kgv::Contexts of the C++ host mirror (include/kgv.hpp), driven by tests/test_gpu_cpp_shared_keycache.py.
// A serial run validates a populated batch twice on one context with its own cache.  Then two std::threads, each on its own context and
// kgv::TransactionValidator, validate the same batch R times at once through one cache, created on the first context and shared with the
// second.  Prints, as plain text for the Python side to compare:
//   serial <status:fee of every transaction>            (one line per pass)
//   thread <t> <status:fee of every transaction>        (one line per call)
//   counters <ecdsa> <lookups> <hits> <inserts> <evictions>
//   shared_keycache_test <dir> <R> <storage_mass_parameter>
// <dir>: txs.bin inputs.bin outputs.bin entries.bin arena.bin (flat records of include/kgv.h).
#include <cstdio>
#include <fstream>
#include <iterator>
#include <mutex>
#include <thread>

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
static std::string verdicts(const std::vector<kgv_tx_result>& r) {
  std::string l;
  for (const auto& x : r) l += " " + std::to_string((int)x.status) + ":" + std::to_string((unsigned long long)x.fee);
  return l;
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: %s <dir> <R> <storage_mass_parameter>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  const int R = std::stoi(argv[2]);
  try {
    kgv::Params p;
    p.storage_mass_parameter = std::stoull(argv[3]);
    kgv::TxBatch b;
    b.assign(slurp<kgv_tx>(dir + "txs.bin"), slurp<kgv_input>(dir + "inputs.bin"), slurp<kgv_output>(dir + "outputs.bin"),
             slurp<kgv_utxo_entry>(dir + "entries.bin"), slurp<uint8_t>(dir + "arena.bin"));
    {
      kgv::Context s(0);
      kgv::KeyCache kc(s, 1 << 12, 1 << 12);
      kgv::TransactionValidator tv(s, p);
      for (int pass = 0; pass < 2; pass++) std::printf("serial%s\n", verdicts(tv.validate_populated_transactions(b, 10)).c_str());
    }
    kgv::Context c0(0), c1(0);
    kgv::KeyCache k0(c0, 1 << 12, 1 << 12);
    kgv::KeyCache k1(c1, k0);
    std::mutex out_mu;
    std::vector<std::string> lines;
    bool failed = false;
    auto body = [&](int t, kgv::Context& c) {
      try {
        kgv::TransactionValidator tv(c, p);
        for (int r = 0; r < R; r++) {
          const std::string l = "thread " + std::to_string(t) + verdicts(tv.validate_populated_transactions(b, 10));
          std::lock_guard<std::mutex> g(out_mu);
          lines.push_back(l);
        }
      } catch (const std::exception& e) {
        std::lock_guard<std::mutex> g(out_mu);
        std::fprintf(stderr, "thread %d: %s\n", t, e.what());
        failed = true;
      }
    };
    std::thread t0(body, 0, std::ref(c0)), t1(body, 1, std::ref(c1));
    t0.join();
    t1.join();
    if (failed) return 1;
    for (const auto& l : lines) std::printf("%s\n", l.c_str());
    for (int e = 0; e < 2; e++) {
      const auto k = k1.counters(e);
      std::printf("counters %d %llu %llu %llu %llu\n", e, (unsigned long long)k.lookups, (unsigned long long)k.hits, (unsigned long long)k.inserts,
                  (unsigned long long)k.evictions);
    }
  } catch (const std::exception& e) {
    std::printf("error %s\n", e.what());
    return 1;
  }
  return 0;
}
