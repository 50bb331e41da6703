// One kgv::UtxoSet shared by two kgv::Contexts of the C++ host mirror (include/kgv.hpp), driven by tests/test_gpu_cpp_shared_utxo.py.  A writer
// thread replays K windows into a view over the set on context A and commits each; after every commit it waits until the reader has
// completed a call that began after it.  A reader thread validates a mempool batch against the committed set through a
// kgv::TransactionValidator of context B, in a loop.  Prints, as plain text for the Python side to compare with its serial run:
//   window <k> <status of every transaction of the window's replay>
//   read <commits completed before the call began> <status of every probe transaction>
//   shared_utxo_mirror_test <dir> <K> <virtual_daa_score> <coinbase_maturity> <storage_mass_parameter>
// <dir>: w<k>_txs.bin w<k>_inputs.bin w<k>_outputs.bin w<k>_arena.bin w<k>_blocks.bin for k < K, and probe_txs.bin probe_inputs.bin
// probe_outputs.bin probe_arena.bin (flat records of include/kgv.h).
#include <atomic>
#include <chrono>
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
static kgv::TxBatch load(const std::string& prefix) {
  kgv::TxBatch b;
  b.assign(slurp<kgv_tx>(prefix + "_txs.bin"), slurp<kgv_input>(prefix + "_inputs.bin"), slurp<kgv_output>(prefix + "_outputs.bin"), {},
           slurp<uint8_t>(prefix + "_arena.bin"));
  return b;
}

int main(int argc, char** argv) {
  if (argc < 6) { std::fprintf(stderr, "usage: %s <dir> <K> <virtual_daa_score> <coinbase_maturity> <storage_mass_parameter>\n", argv[0]); return 2; }
  const std::string dir = std::string(argv[1]) + "/";
  const int K = std::stoi(argv[2]);
  const uint64_t vdaa = std::stoull(argv[3]);
  try {
    kgv::Params p;
    p.coinbase_maturity = std::stoull(argv[4]);
    p.storage_mass_parameter = std::stoull(argv[5]);
    std::vector<kgv::TxBatch> windows;
    std::vector<std::vector<kgv_replay_block>> blocks;
    for (int k = 0; k < K; k++) {
      const std::string w = dir + "w" + std::to_string(k);
      windows.push_back(load(w));
      blocks.push_back(slurp<kgv_replay_block>(w + "_blocks.bin"));
    }
    const kgv::TxBatch probe = load(dir + "probe");
    kgv::Context a(0), b(0);
    kgv::UtxoSet base(a, 1 << 13);
    kgv::UtxoSet view(a, base, 1 << 12);
    kgv::TransactionValidator tv_a(a, p), tv_b(b, p);

    std::atomic<int> commits{0}, done_after{-1};
    std::atomic<bool> stop{false}, failed{false};
    std::mutex out_mu;
    std::vector<std::string> lines;
    std::thread reader([&] {
      try {
        while (!stop.load()) {
          const int began = commits.load();
          auto r = tv_b.validate_mempool_transactions_in_utxo_context(base, probe, vdaa);
          std::string l = "read " + std::to_string(began);
          for (const auto& x : r.results) l += " " + std::to_string((int)x.status);
          {
            std::lock_guard<std::mutex> g(out_mu);
            lines.push_back(l);
          }
          done_after.store(began);
        }
      } catch (const std::exception& e) {
        std::fprintf(stderr, "reader: %s\n", e.what());
        failed.store(true);
      }
    });
    // waits with a deadline: a hang fails the run instead of blocking it
    auto wait_reader = [&](int c) {
      const auto t0 = std::chrono::steady_clock::now();
      while (done_after.load() < c && !failed.load()) {
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(120)) throw std::runtime_error("timed out waiting for the reader");
        std::this_thread::sleep_for(std::chrono::microseconds(200));
      }
    };
    std::thread writer([&] {
      try {
        wait_reader(0);
        for (int k = 0; k < K; k++) {
          auto res = tv_a.replay_window(view, windows[k], blocks[k]);
          view.commit();
          std::string l = "window " + std::to_string(k);
          for (const auto& x : res) l += " " + std::to_string((int)x.status);
          {
            std::lock_guard<std::mutex> g(out_mu);
            lines.push_back(l);
          }
          commits.store(k + 1);
          wait_reader(k + 1);
        }
      } catch (const std::exception& e) {
        std::fprintf(stderr, "writer: %s\n", e.what());
        failed.store(true);
      }
      stop.store(true);
    });
    writer.join();
    reader.join();
    for (const auto& l : lines) std::printf("%s\n", l.c_str());
    if (failed.load()) return 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  return 0;
}
