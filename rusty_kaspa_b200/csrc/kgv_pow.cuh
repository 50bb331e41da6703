// kgv_pow.cuh — the per-header pieces of header validation in isolation (kgv_headers.cu), host-compilable (KGV_HD):
// tests/hostsim/hostsim_pow.cpp builds the same functions with g++.
//
// Restates:
//   hashing::header::hash_override_nonce_time   consensus/core/src/hashing/header.rs:7-30 (keyed BLAKE2b "BlockHash"; blue work as
//                                               write_var_bytes of its big-endian bytes without leading zeros, hashing/mod.rs:76-86)
//   XoShiRo256PlusPlus                          consensus/pow/src/xoshiro.rs
//   Matrix::rand_matrix_no_rank_check           consensus/pow/src/matrix.rs:113-125 (16 nibbles per draw, low nibble first)
//   Matrix::compute_rank                        matrix.rs:141-174, operation for operation in IEEE double without contraction
//   Matrix::heavy_hash                          matrix.rs:176-200
//   Uint256::from_compact_target_bits           math/src/lib.rs:64-79 with the shift of math/src/uint.rs:67-84
//   calc_level_from_pow                         consensus/pow/src/lib.rs:72-75
//
// compute_rank is the one place where the order of floating-point operations decides a result: a rank below 64 makes Matrix::generate
// draw another matrix.  Every element a[k][p] sees the same sequence of divisions, products and differences as in the reference: the
// pivot row's division, then for every other row with |a[k][i]| > 1e-9 the update a[k][p] -= a[j][p] * a[k][i].  The products and
// differences are separate roundings (__dmul_rn / __dsub_rn on the device; the host build has no FMA to contract into), as in Rust.
// Columns are independent within one pivot step, so the device spreads them over threads (rank_column); the host build walks them in
// order.  Either way each element's operations are the reference's.
#pragma once
#include "../../include/kgv.h"
#include "kgv_keccak.cuh"
#include "kgv_muhash.cuh"  // b2b_init_keyed_words

#if !defined(__CUDACC__)
#include <cmath>
#include <cstring>
#endif

namespace kgv {

constexpr double RANK_EPS = 1e-9;
constexpr int RANK_STRIDE = 65;  // row pitch of the f64 matrix, in doubles (one spare column keeps the pivot search off one bank)

#if defined(__CUDACC__)
KGV_HD double f64_div(double a, double b) { return __ddiv_rn(a, b); }
KGV_HD double f64_mul(double a, double b) { return __dmul_rn(a, b); }
KGV_HD double f64_sub(double a, double b) { return __dsub_rn(a, b); }
KGV_HD uint64_t ld_u64(const uint8_t* p) { return *(const uint64_t*)p; }  // 8-byte aligned by the callers' contract
#else
inline double f64_div(double a, double b) { return a / b; }
inline double f64_mul(double a, double b) { return a * b; }
inline double f64_sub(double a, double b) { return a - b; }
inline uint64_t ld_u64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
#endif

// ---- block hash -------------------------------------------------------------------------------------------------------------------

// keyed BLAKE2b "BlockHash" (crypto/hashes/src/hashers.rs:27), the key as two little-endian words (no local key array, DESIGN.md §6)
KGV_HD void b2b_init_block_hash(Blake2b& h) { b2b_init_keyed_words(h, 0x7361486b636f6c42ull, 0x0000000000000068ull, 9); }

// one u64 at any byte position of the block buffer: two word ORs instead of eight byte steps
KGV_HD void b2b_u64_any(Blake2b& s, uint64_t v) {
  const uint32_t r = s.fill & 7;
  if (r == 0 || s.fill + 8 > 128) {
    if (r == 0) { b2b_u64(s, v); return; }
#pragma unroll 1
    for (int i = 0; i < 8; i++) b2b_byte(s, (uint32_t)(v >> (8 * i)));
    return;
  }
  s.m[s.fill >> 3] |= v << (8 * r);
  s.m[(s.fill >> 3) + 1] |= v >> (64 - 8 * r);
  s.fill += 8;
  s.t += 8;
  s.fresh = false;
}

// Both callers have checked the arena ranges.  parents: the header's first parent hash; lens: its level sizes.
KGV_HD void header_hash(const kgv_header& h, const uint8_t* parents, const uint32_t* lens, uint64_t nonce, uint64_t timestamp, uint64_t* out4) {
  Blake2b s;
  b2b_init_block_hash(s);
  b2b_u16(s, h.version);
  b2b_u64_any(s, h.n_levels);
  for (uint32_t l = 0; l < h.n_levels; l++) {
    const uint32_t np = lens[l];
    b2b_u64_any(s, np);
    for (uint32_t k = 0; k < np; k++, parents += 32) {
#pragma unroll
      for (int w = 0; w < 4; w++) b2b_u64_any(s, ld_u64(parents + 8 * w));
    }
  }
  const uint8_t* roots = h.hash_merkle_root;  // hash_merkle_root, accepted_id_merkle_root, utxo_commitment: 96 contiguous bytes
#pragma unroll 1
  for (int w = 0; w < 12; w++) b2b_u64_any(s, ld_u64(roots + 8 * w));
  b2b_u64_any(s, timestamp);
  b2b_u32(s, h.bits);
  b2b_u64_any(s, nonce);
  b2b_u64_any(s, h.daa_score);
  b2b_u64_any(s, h.blue_score);
  uint32_t z = 0;
  while (z < 24 && h.blue_work[z] == 0) z++;
  b2b_u64_any(s, 24 - z);
  for (uint32_t k = z; k < 24; k++) b2b_byte(s, h.blue_work[k]);
#pragma unroll 1
  for (int w = 0; w < 4; w++) b2b_u64_any(s, ld_u64(h.pruning_point + 8 * w));
  b2b_final(s, out4);
}

// levels_off / parents_off ranges inside the arena; on success *n_par = the header's parents over all levels
KGV_HD bool header_ranges_ok(const kgv_header& h, const uint32_t* level_len, uint64_t n_level_entries, uint64_t n_parents, uint64_t* n_par) {
  if ((uint64_t)h.levels_off + h.n_levels > n_level_entries) return false;
  uint64_t tot = 0;
  for (uint32_t l = 0; l < h.n_levels; l++) tot += level_len[h.levels_off + l];
  if (h.parents_off > n_parents || tot > n_parents - h.parents_off) return false;
  *n_par = tot;
  return true;
}

// ---- matrix -----------------------------------------------------------------------------------------------------------------------

struct Xoshiro {
  uint64_t s0, s1, s2, s3;
};
KGV_HD void xoshiro_seed(Xoshiro& x, const uint64_t* w4) { x.s0 = w4[0]; x.s1 = w4[1]; x.s2 = w4[2]; x.s3 = w4[3]; }
KGV_HD uint64_t xoshiro_next(Xoshiro& x) {
  const uint64_t res = x.s0 + rotl64(x.s0 + x.s3, 23);
  const uint64_t t = x.s1 << 17;
  x.s2 ^= x.s0;
  x.s3 ^= x.s1;
  x.s1 ^= x.s2;
  x.s0 ^= x.s3;
  x.s2 ^= t;
  x.s3 = rotl64(x.s3, 45);
  return res;
}
// 64 rows x 4 draws: element (r, 16q + s) = (w[4r + q] >> 4s) & 15
KGV_HD void matrix_draw(Xoshiro& x, uint64_t* w256) {
  for (int i = 0; i < 256; i++) w256[i] = xoshiro_next(x);
}
KGV_HD uint32_t matrix_elem(const uint64_t* w256, int r, int c) { return (uint32_t)(w256[4 * r + (c >> 4)] >> (4 * (c & 15))) & 15u; }

// column p of pivot step i with pivot row j: the division of a[j][p], then every other row's update, in the reference's row order.
// Rows go in blocks of 16, all loads of a block before its stores: the compiler cannot tell column i from column p, so a load after a
// store would wait for it.  A row that the reference skips (k == j, or |a[k][i]| <= eps) gets its own value back.
constexpr int RANK_ROWS = 16;
KGV_HD void rank_column(double* a, int i, int j, int p) {
  const double ajp = f64_div(a[j * RANK_STRIDE + p], a[j * RANK_STRIDE + i]);
  a[j * RANK_STRIDE + p] = ajp;
  for (int k0 = 0; k0 < 64; k0 += RANK_ROWS) {
    double ki[RANK_ROWS], kp[RANK_ROWS];
#pragma unroll
    for (int q = 0; q < RANK_ROWS; q++) {
      ki[q] = a[(k0 + q) * RANK_STRIDE + i];
      kp[q] = a[(k0 + q) * RANK_STRIDE + p];
    }
#pragma unroll
    for (int q = 0; q < RANK_ROWS; q++) {
      const bool upd = k0 + q != j && fabs(ki[q]) > RANK_EPS;
      const double v = f64_sub(kp[q], f64_mul(ajp, ki[q]));
      a[(k0 + q) * RANK_STRIDE + p] = upd ? v : kp[q];
    }
  }
}

// the whole of compute_rank on one thread (host build): a is 64 rows of RANK_STRIDE doubles, overwritten
KGV_HD uint32_t rank_serial(double* a) {
  uint64_t sel = 0;
  uint32_t rank = 0;
  for (int i = 0; i < 64; i++) {
    int j = 0;
    while (j < 64 && !(!((sel >> j) & 1) && fabs(a[j * RANK_STRIDE + i]) > RANK_EPS)) j++;
    if (j == 64) continue;
    rank++;
    sel |= 1ull << j;
    for (int p = i + 1; p < 64; p++) rank_column(a, i, j, p);
  }
  return rank;
}

KGV_HD void matrix_to_f64(const uint64_t* w256, double* a) {
  for (int e = 0; e < 64 * 64; e++) a[(e >> 6) * RANK_STRIDE + (e & 63)] = (double)matrix_elem(w256, e >> 6, e & 63);
}

// Matrix::generate on one thread (host build): src.draw(w256) yields the next candidate matrix; returns the number drawn.  The device runs
// the same loop with the rank spread over a CTA (cta_generate, kgv_headers.cu).
template <class Source>
KGV_HD uint32_t matrix_generate_serial(Source& src, uint64_t* w256, double* a) {
  for (uint32_t tries = 1;; tries++) {
    src.draw(w256);
    matrix_to_f64(w256, a);
    if (rank_serial(a) == 64) return tries;
  }
}
struct XoshiroSource {
  Xoshiro x;
  KGV_HD void draw(uint64_t* w256) { matrix_draw(x, w256); }
};

// the product of matrix_draw's matrix and the nibble vector of h (high nibble first), folded back to 32 bytes, XORed with h and hashed
// with cSHAKE256 "HeavyHash".  rows[r] = sum_j m[r][j] * vec[j] (u16, wrapping as in the reference; nibbles keep it below 2^14).
KGV_HD uint32_t heavy_row_sum(const uint64_t* w256, int r, const uint64_t* h4) {
  uint32_t sum = 0;
  for (int c = 0; c < 64; c++) {
    const uint32_t byte = (uint32_t)(h4[c >> 4] >> (8 * ((c >> 1) & 7))) & 0xFF;
    const uint32_t v = (c & 1) ? (byte & 15) : (byte >> 4);
    sum += matrix_elem(w256, r, c) * v;
  }
  return sum & 0xFFFF;
}
KGV_HD void heavy_finish(const uint32_t* rows64, const uint64_t* h4, uint64_t* out4) {
  uint64_t p[4] = {0, 0, 0, 0};
  for (int i = 0; i < 32; i++) {
    const uint64_t b = ((rows64[2 * i] >> 10) << 4 | (rows64[2 * i + 1] >> 10)) & 0xFF;
    p[i >> 3] |= b << (8 * (i & 7));
  }
  for (int w = 0; w < 4; w++) p[w] ^= h4[w];
  kheavy_hash(p, out4);
}

// ---- target and level -------------------------------------------------------------------------------------------------------------

// Uint256::from_compact_target_bits.  A release build of Uint256 << s shifts by s mod 256 (overflowing_shl: s %= BITS), so exponents past
// 34 wrap around rather than giving zero; bits shifted past 2^256 are lost.
KGV_HD void compact_target(uint32_t bits, uint64_t* t4) {
  const uint32_t e = bits >> 24;
  uint32_t mant, sh;
  if (e <= 3) { mant = (bits & 0xFFFFFF) >> (8 * (3 - e)); sh = 0; }
  else { mant = bits & 0xFFFFFF; sh = 8 * (e - 3); }
  t4[0] = t4[1] = t4[2] = t4[3] = 0;
  if (mant > 0x7FFFFF) return;
  sh &= 255;
  const uint32_t wq = sh >> 6, r = sh & 63;
  t4[wq] = (uint64_t)mant << r;
  if (r && wq < 3) t4[wq + 1] = (uint64_t)mant >> (64 - r);
}
KGV_HD bool u256_le(const uint64_t* a, const uint64_t* b) {
  for (int w = 3; w >= 0; w--)
    if (a[w] != b[w]) return a[w] < b[w];
  return true;
}
KGV_HD uint32_t u256_bits(const uint64_t* a) {
  for (int w = 3; w >= 0; w--)
    if (a[w]) {
#if defined(__CUDACC__)
      return 64 * w + 64 - __clzll((long long)a[w]);
#else
      return 64 * w + 64 - __builtin_clzll(a[w]);
#endif
    }
  return 0;
}
KGV_HD uint32_t level_from_pow(const uint64_t* pow4, uint32_t max_block_level) {
  const int64_t l = (int64_t)max_block_level - (int64_t)u256_bits(pow4);
  return l > 0 ? (uint32_t)l : 0u;
}

// ---- the isolation rules ----------------------------------------------------------------------------------------------------------

// validate_header_in_isolation's order; direct: level-0 parent hashes (n_direct of them)
KGV_HD void header_rules(const kgv_header& h, const uint8_t* direct, uint32_t n_direct, const kgv_header_rules& r, bool passed, kgv_header_result& out) {
  out.a = out.b = 0;
  if (h.version != r.block_version) { out.status = KGV_HEADER_WRONG_BLOCK_VERSION; out.a = h.version; return; }
  const uint64_t max_time = r.now_ms + r.timestamp_deviation_tolerance * 1000;  // u64 arithmetic wraps, as the reference's release build
  if (h.timestamp > max_time) { out.status = KGV_HEADER_TIME_TOO_FAR_INTO_THE_FUTURE; out.a = h.timestamp; out.b = max_time; return; }
  if (n_direct == 0) { out.status = KGV_HEADER_NO_PARENTS; return; }
  if (n_direct > r.max_block_parents) { out.status = KGV_HEADER_TOO_MANY_PARENTS; out.a = n_direct; out.b = r.max_block_parents; return; }
  for (uint32_t k = 0; k < n_direct; k++) {
    bool origin = true;
    for (int w = 0; w < 4; w++) origin &= ld_u64(direct + 32 * k + 8 * w) == 0xFEFEFEFEFEFEFEFEull;
    if (origin) { out.status = KGV_HEADER_ORIGIN_PARENT; return; }
  }
  out.status = (passed || (r.flags & KGV_HEADER_SKIP_POW)) ? KGV_HEADER_OK : KGV_HEADER_INVALID_POW;
}

}  // namespace kgv
