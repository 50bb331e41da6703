// Host build of the device script engine (kgv_script_dev.cuh) for GPU-less tests (TEST BUILD ONLY).  The harness drives it round
// by round exactly as kgv_scripts_dev.cu does: run the input from the start over its verdict log, answer the one request, repeat.
#include "../../rusty_kaspa_b200/csrc/kgv_script_dev.cuh"
#include <cstring>
#include <memory>
#include <vector>
using namespace kgv;

typedef int (*exec_fn)(const kgv_tx_batch*, uint32_t, uint32_t, kgv_verdict_fn, void*, uint8_t*);

static std::vector<DevEntry> dev_entries(const kgv_tx_batch* b) {
  std::vector<DevEntry> v(b->n_inputs);
  for (size_t i = 0; i < b->n_inputs; i++) {
    const kgv_utxo_entry& e = b->entries[i];
    v[i] = DevEntry{e.amount, e.block_daa_score, b->bytes + e.script_off, e.script_len, e.spk_version, e.is_coinbase, (uint8_t)(e.pad_[0] ? 0 : 1)};
  }
  return v;
}
static void log_set(uint8_t* log, uint32_t k, uint32_t v) { log[k >> 2] = (uint8_t)((log[k >> 2] & ~(3u << (2 * (k & 3)))) | ((v & 3) << (2 * (k & 3)))); }

// A deterministic stand-in for signature verification, the same for both engines.  mode 0: a hash of (input, kind, hash type, key, sig)
// picks VALID / INVALID / PK_PARSE_ERR / SIG_PARSE_ERR (5:3:1:1); mode 1: VALID iff the key's first byte is 0xAA, else INVALID.
static int fake_verdict(int mode, uint32_t in_abs, uint32_t ecdsa, uint32_t hash_type, const uint8_t* key, const uint8_t* sig) {
  const uint32_t kl = ecdsa ? 33 : 32;
  if (mode == 1) return key[0] == 0xAA ? KGV_SIG_VALID : KGV_SIG_INVALID;
  uint64_t h = 1469598103934665603ull ^ ((uint64_t)in_abs << 16) ^ (ecdsa << 8) ^ hash_type;
  for (uint32_t i = 0; i < kl; i++) h = (h ^ key[i]) * 1099511628211ull;
  for (uint32_t i = 0; i < 64; i++) h = (h ^ sig[i]) * 1099511628211ull;
  const uint32_t r = (uint32_t)((h >> 29) % 10);
  return r < 5 ? KGV_SIG_VALID : r < 8 ? KGV_SIG_INVALID : r < 9 ? KGV_SIG_PK_PARSE_ERR : KGV_SIG_SIG_PARSE_ERR;
}
struct HostCb { int mode; };
static int host_cb(void* user, const kgv_sig_request* r) {
  return fake_verdict(((HostCb*)user)->mode, r->input, r->ecdsa, r->hash_type, r->key, r->sig);
}

extern "C" {
uint32_t hs_slot_bytes() { return (uint32_t)sizeof(ScriptSlot); }

// One pass of one input over the verdicts given so far.  Returns a KGV_SCRIPT_* code, or 254 with the request in req_out
// (hash_type, ecdsa, key[33], sig[64] = 99 bytes).
int hs_script_run(const kgv_tx_batch* b, uint32_t tx, uint32_t input_index, const uint8_t* verdicts, uint32_t n_verdicts, uint8_t* req_out) {
  std::vector<DevEntry> de = dev_entries(b);
  BatchView v{b->txs, b->inputs, b->outputs, de.data(), b->bytes};
  std::unique_ptr<ScriptSlot> slot(new ScriptSlot());
  uint8_t log[SE_LOG_BYTES] = {0};
  for (uint32_t k = 0; k < n_verdicts && k < 4 * SE_LOG_BYTES; k++) log_set(log, k, verdicts[k]);
  ScriptReq rq;
  memset(&rq, 0, sizeof rq);
  const uint8_t r = script_run_input(v, tx, b->txs[tx].first_input + input_index, slot.get(), log, n_verdicts, &rq);
  if (r == SE_NEEDS && req_out) { req_out[0] = rq.hash_type; req_out[1] = rq.ecdsa; memcpy(req_out + 2, rq.key, 33); memcpy(req_out + 35, rq.sig, 64); }
  return r;
}

// Every input of every tx through both engines with the same fake verdicts: dev_out / host_out get the KGV_SCRIPT_* codes,
// checks_out the device engine's signature checks per input.  host_exec = kgv_script_execute of libkgv.so.
int hs_compare(const kgv_tx_batch* b, exec_fn host_exec, int mode, uint8_t* dev_out, uint8_t* host_out, uint32_t* checks_out) {
  std::vector<DevEntry> de = dev_entries(b);
  BatchView v{b->txs, b->inputs, b->outputs, de.data(), b->bytes};
  std::unique_ptr<ScriptSlot> slot(new ScriptSlot());
  HostCb cb{mode};
  for (uint32_t t = 0; t < b->n_txs; t++) {
    for (uint32_t k = 0; k < b->txs[t].n_inputs; k++) {
      const uint32_t in_abs = b->txs[t].first_input + k;
      uint8_t log[SE_LOG_BYTES] = {0};
      uint32_t n = 0;
      uint8_t r;
      for (;;) {
        ScriptReq rq;
        memset(&rq, 0, sizeof rq);
        r = script_run_input(v, t, in_abs, slot.get(), log, n, &rq);
        if (r != SE_NEEDS) break;
        if (n >= 4 * SE_LOG_BYTES) return -1;
        log_set(log, n, (uint32_t)fake_verdict(mode, in_abs, rq.ecdsa, rq.hash_type, rq.key, rq.sig));
        n++;
      }
      dev_out[in_abs] = r;
      checks_out[in_abs] = n;
      if (host_exec(b, t, k, host_cb, &cb, &host_out[in_abs]) != 0) return -2;
    }
  }
  return 0;
}
}
