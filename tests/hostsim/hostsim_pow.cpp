// Host build of the per-header code of kgv_validate_headers_in_isolation (kgv_pow.cuh, kgv_keccak.cuh) for GPU-less tests (TEST BUILD
// ONLY): the same functions k_header_hash / k_header_validate call, with the rank walked column by column on one thread.
#include <vector>

#include "../../rusty_kaspa_b200/csrc/kgv_pow.cuh"
using namespace kgv;

static void put32(uint8_t* o, const uint64_t* w) {
  for (int k = 0; k < 32; k++) o[k] = (uint8_t)(w[k / 8] >> (8 * (k % 8)));
}
static void get32(uint64_t* w, const uint8_t* in) {
  for (int k = 0; k < 4; k++) w[k] = ld_u64(in + 8 * k);
}
static void pack(const uint8_t* m4096, uint64_t* w256) {
  for (int i = 0; i < 256; i++) w256[i] = 0;
  for (int e = 0; e < 4096; e++) w256[4 * (e >> 6) + ((e & 63) >> 4)] |= (uint64_t)(m4096[e] & 15) << (4 * (e & 15));
}

// a candidate source that yields caller matrices in turn (the retry loop with rank-deficient candidates)
struct ScriptedSource {
  const uint8_t* mats;
  uint32_t n, next;
  void draw(uint64_t* w256) { pack(mats + 4096 * (next < n ? next : n - 1), w256); next++; }
};

extern "C" {
void hs_keccak_f1600(uint64_t* st25) { keccak_f1600(st25); }
void hs_pow_hash(const uint8_t* pre32, uint64_t timestamp, uint64_t nonce, uint8_t* out32) {
  uint64_t p[4], o[4];
  get32(p, pre32);
  pow_hash(p, timestamp, nonce, o);
  put32(out32, o);
}
// header hash with the given nonce / timestamp (the header's own for the block hash, 0 / 0 for the pre-PoW hash); parents32 / level_len:
// the arena, as the kernels read it
void hs_header_hash(const kgv_header* h, const uint8_t* parents32, const uint32_t* level_len, uint64_t nonce, uint64_t timestamp, uint8_t* out32) {
  uint64_t d[4];
  header_hash(*h, parents32 + 32 * h->parents_off, level_len + h->levels_off, nonce, timestamp, d);
  put32(out32, d);
}
// compute_rank of a 64 x 64 u16 matrix
uint32_t hs_rank(const uint16_t* m) {
  std::vector<double> a(64 * RANK_STRIDE);
  for (int e = 0; e < 4096; e++) a[(e >> 6) * RANK_STRIDE + (e & 63)] = (double)m[e];
  return rank_serial(a.data());
}
// Matrix::generate from a 32-byte seed: 4096 nibbles out; returns the matrices drawn
uint32_t hs_generate(const uint8_t* seed32, uint8_t* out4096) {
  XoshiroSource src;
  uint64_t s[4], w[256];
  get32(s, seed32);
  xoshiro_seed(src.x, s);
  std::vector<double> a(64 * RANK_STRIDE);
  const uint32_t tries = matrix_generate_serial(src, w, a.data());
  for (int e = 0; e < 4096; e++) out4096[e] = (uint8_t)matrix_elem(w, e >> 6, e & 63);
  return tries;
}
// the generate loop over n caller candidates (4096 nibbles each, the last repeated): the accepted one out, returns the candidates drawn
uint32_t hs_generate_scripted(const uint8_t* mats, uint32_t n, uint8_t* out4096) {
  ScriptedSource src{mats, n, 0};
  uint64_t w[256];
  std::vector<double> a(64 * RANK_STRIDE);
  const uint32_t tries = matrix_generate_serial(src, w, a.data());
  for (int e = 0; e < 4096; e++) out4096[e] = (uint8_t)matrix_elem(w, e >> 6, e & 63);
  return tries;
}
// Matrix::heavy_hash with a caller matrix (4096 nibbles)
void hs_heavy_hash(const uint8_t* m4096, const uint8_t* in32, uint8_t* out32) {
  uint64_t w[256], h[4], o[4];
  uint32_t rows[64];
  pack(m4096, w);
  get32(h, in32);
  for (int r = 0; r < 64; r++) rows[r] = heavy_row_sum(w, r, h);
  heavy_finish(rows, h, o);
  put32(out32, o);
}
void hs_compact_target(uint32_t bits, uint8_t* out32) {
  uint64_t t[4];
  compact_target(bits, t);
  put32(out32, t);
}
// the whole of k_header_validate for one header of an arena (ranges already checked by the caller)
void hs_validate(const kgv_header* h, const uint8_t* parents32, const uint32_t* level_len, const kgv_header_rules* r, kgv_header_result* res,
                 uint8_t* pow32, uint8_t* pre32) {
  const uint8_t* parents = parents32 + 32 * h->parents_off;
  const uint32_t* lens = level_len + h->levels_off;
  uint64_t pre[4], ph[4], w[256], pw[4], target[4];
  uint32_t rows[64];
  header_hash(*h, parents, lens, 0, 0, pre);
  pow_hash(pre, h->timestamp, h->nonce, ph);
  XoshiroSource src;
  xoshiro_seed(src.x, pre);
  std::vector<double> a(64 * RANK_STRIDE);
  matrix_generate_serial(src, w, a.data());
  for (int t = 0; t < 64; t++) rows[t] = heavy_row_sum(w, t, ph);
  heavy_finish(rows, ph, pw);
  compact_target(h->bits, target);
  const bool genesis = h->n_levels == 0;
  const bool passed = genesis || u256_le(pw, target);
  header_rules(*h, parents, genesis ? 0u : lens[0], *r, passed, *res);
  res->level = (uint8_t)(genesis ? r->max_block_level : level_from_pow(pw, r->max_block_level));
  res->pow_passed = passed;
  res->pad_ = 0;
  put32(pow32, pw);
  put32(pre32, pre);
}
}
