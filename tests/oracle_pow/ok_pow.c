/* ok_pow.c — C restatement of header validation in isolation (TEST INFRASTRUCTURE: the checker of kgv_validate_headers_in_isolation and
 * kgv_hash_headers, never the thing under test).  Written from the reference's Rust and the public specifications, independently of
 * the device code:
 *   consensus/core/src/hashing/header.rs:7-35              header serialization, keyed BLAKE2b-256 "BlockHash" (RFC 7693)
 *   crypto/hashes/src/pow_hashers.rs                       cSHAKE256 "ProofOfWorkHash" / "HeavyHash" (NIST SP 800-185), built here
 *                                                          by absorbing the bytepad block, not from constants
 *   consensus/pow/src/xoshiro.rs, matrix.rs                xoshiro256++, generate, compute_rank, heavy_hash
 *   math/src/lib.rs:64-79, math/src/uint.rs:67-84          from_compact_target_bits, with the shift taken modulo 256
 *   consensus/pow/src/lib.rs:56-75                         calc_block_level_check_pow, calc_level_from_pow
 *   consensus/src/pipeline/header_processor/pre_ghostdag_validation.rs:17-68,102-106   the rules, in order
 * Record layouts are those of include/kgv.h (kgv_header, kgv_header_rules, kgv_header_result), restated below.
 * Built by __graft_entry__.build() (or the test fixture) into tests/oracle_pow/libok_pow.so. */
#include <math.h>
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

typedef struct {
  uint8_t hash_merkle_root[32], accepted_id_merkle_root[32], utxo_commitment[32], pruning_point[32], blue_work[24];
  uint64_t timestamp, nonce, daa_score, blue_score, parents_off;
  uint32_t levels_off, n_levels, bits;
  uint16_t version, pad_;
} ok_header;
typedef struct {
  uint64_t timestamp_deviation_tolerance, now_ms;
  uint32_t block_version, max_block_parents, max_block_level, flags;
} ok_header_rules;
typedef struct {
  uint32_t status;
  uint8_t level, pow_passed;
  uint16_t pad_;
  uint64_t a, b;
} ok_header_result;
_Static_assert(sizeof(ok_header) == 208, "layout of kgv_header");
_Static_assert(sizeof(ok_header_rules) == 32, "layout of kgv_header_rules");
_Static_assert(sizeof(ok_header_result) == 24, "layout of kgv_header_result");

/* ---- BLAKE2b-256, keyed (RFC 7693) ---- */
static const uint64_t B2_IV[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                  0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
static const uint8_t B2_SIGMA[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
typedef struct {
  uint64_t h[8], t;
  uint8_t buf[128];
  size_t n;
} b2;
static uint64_t rd64(const uint8_t* p) {
  uint64_t v;
  memcpy(&v, p, 8);
  return v;
}
static uint64_t ror(uint64_t x, int r) { return (x >> r) | (x << (64 - r)); }
static void b2_compress(b2* s, int last) {
  uint64_t v[16], m[16];
  for (int i = 0; i < 16; i++) m[i] = rd64(s->buf + 8 * i);
  for (int i = 0; i < 8; i++) { v[i] = s->h[i]; v[i + 8] = B2_IV[i]; }
  v[12] ^= s->t;
  if (last) v[14] = ~v[14];
#define G(a, b, c, d, x, y) \
  v[a] += v[b] + x; v[d] = ror(v[d] ^ v[a], 32); v[c] += v[d]; v[b] = ror(v[b] ^ v[c], 24); \
  v[a] += v[b] + y; v[d] = ror(v[d] ^ v[a], 16); v[c] += v[d]; v[b] = ror(v[b] ^ v[c], 63);
  for (int r = 0; r < 12; r++) {
    const uint8_t* z = B2_SIGMA[r];
    G(0, 4, 8, 12, m[z[0]], m[z[1]]) G(1, 5, 9, 13, m[z[2]], m[z[3]]) G(2, 6, 10, 14, m[z[4]], m[z[5]]) G(3, 7, 11, 15, m[z[6]], m[z[7]])
    G(0, 5, 10, 15, m[z[8]], m[z[9]]) G(1, 6, 11, 12, m[z[10]], m[z[11]]) G(2, 7, 8, 13, m[z[12]], m[z[13]]) G(3, 4, 9, 14, m[z[14]], m[z[15]])
  }
#undef G
  for (int i = 0; i < 8; i++) s->h[i] ^= v[i] ^ v[i + 8];
}
static void b2_update(b2* s, const void* data, size_t len) {
  const uint8_t* p = data;
  while (len) {
    if (s->n == 128) { s->t += 128; b2_compress(s, 0); s->n = 0; }
    size_t k = 128 - s->n < len ? 128 - s->n : len;
    memcpy(s->buf + s->n, p, k);
    s->n += k; p += k; len -= k;
  }
}
static void b2_init_key(b2* s, const char* key) {
  size_t kl = strlen(key);
  memcpy(s->h, B2_IV, 64);
  s->h[0] ^= 0x01010000ULL ^ (kl << 8) ^ 32;
  s->t = 0;
  memset(s->buf, 0, 128);
  memcpy(s->buf, key, kl);
  s->n = 128;
}
static void b2_final(b2* s, uint8_t out[32]) {
  s->t += s->n;
  memset(s->buf + s->n, 0, 128 - s->n);
  b2_compress(s, 1);
  memcpy(out, s->h, 32);
}
static void u64le(b2* s, uint64_t v) { b2_update(s, &v, 8); }

void ok_pow_header_hash(const ok_header* h, const uint8_t* parents32, const uint32_t* level_len, uint64_t nonce, uint64_t timestamp, uint8_t out[32]) {
  b2 s;
  b2_init_key(&s, "BlockHash");
  b2_update(&s, &h->version, 2);
  u64le(&s, h->n_levels);
  const uint8_t* p = parents32 + 32 * h->parents_off;
  for (uint32_t l = 0; l < h->n_levels; l++) {
    uint32_t np = level_len[h->levels_off + l];
    u64le(&s, np);
    b2_update(&s, p, 32 * (size_t)np);
    p += 32 * (size_t)np;
  }
  b2_update(&s, h->hash_merkle_root, 32);
  b2_update(&s, h->accepted_id_merkle_root, 32);
  b2_update(&s, h->utxo_commitment, 32);
  u64le(&s, timestamp);
  b2_update(&s, &h->bits, 4);
  u64le(&s, nonce);
  u64le(&s, h->daa_score);
  u64le(&s, h->blue_score);
  int z = 0;
  while (z < 24 && !h->blue_work[z]) z++;
  u64le(&s, 24 - z);
  b2_update(&s, h->blue_work + z, 24 - z);
  b2_update(&s, h->pruning_point, 32);
  b2_final(&s, out);
}

/* ---- Keccak-f1600 and cSHAKE256 ---- */
static const uint64_t KRC[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL, 0x000000000000808BULL, 0x0000000080000001ULL,
    0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008AULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000AULL,
    0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL, 0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL,
    0x000000000000800AULL, 0x800000008000000AULL, 0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
static const int KROT[5][5] = {{0, 36, 3, 41, 18}, {1, 44, 10, 45, 2}, {62, 6, 43, 15, 61}, {28, 55, 25, 21, 56}, {27, 20, 39, 8, 14}};
static uint64_t rol(uint64_t v, int r) { return r ? (v << r) | (v >> (64 - r)) : v; }
void ok_keccak_f1600(uint64_t a[25]) {
  for (int rnd = 0; rnd < 24; rnd++) {
    uint64_t c[5], b[25];
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    for (int x = 0; x < 5; x++) {
      uint64_t d = c[(x + 4) % 5] ^ rol(c[(x + 1) % 5], 1);
      for (int y = 0; y < 5; y++) a[x + 5 * y] ^= d;
    }
    for (int x = 0; x < 5; x++)
      for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rol(a[x + 5 * y], KROT[x][y]);
    for (int y = 0; y < 5; y++)
      for (int x = 0; x < 5; x++) a[x + 5 * y] = b[x + 5 * y] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);
    a[0] ^= KRC[rnd];
  }
}
/* cSHAKE256(msg, 256 bits, N = "", S = custom) for msg_len < 136 */
static void cshake256(const char* custom, const uint8_t* msg, size_t msg_len, uint8_t out[32]) {
  uint8_t blk[136];
  uint64_t a[25];
  memset(a, 0, sizeof a);
  size_t sl = strlen(custom), k = 0;
  memset(blk, 0, 136);
  blk[k++] = 1; blk[k++] = 136;      /* left_encode(136) */
  blk[k++] = 1; blk[k++] = 0;        /* encode_string(""): left_encode(0) */
  blk[k++] = 1; blk[k++] = (uint8_t)(8 * sl);  /* encode_string(S): left_encode(8 |S|), S < 32 bytes */
  memcpy(blk + k, custom, sl);
  for (int i = 0; i < 17; i++) a[i] ^= rd64(blk + 8 * i);
  ok_keccak_f1600(a);
  memset(blk, 0, 136);
  memcpy(blk, msg, msg_len);
  blk[msg_len] ^= 0x04;
  blk[135] ^= 0x80;
  for (int i = 0; i < 17; i++) a[i] ^= rd64(blk + 8 * i);
  ok_keccak_f1600(a);
  memcpy(out, a, 32);
}

/* ---- matrix ---- */
typedef struct { uint64_t s[4]; } xo;
static uint64_t xo_next(xo* x) {
  uint64_t r = x->s[0] + rol(x->s[0] + x->s[3], 23), t = x->s[1] << 17;
  x->s[2] ^= x->s[0]; x->s[3] ^= x->s[1]; x->s[1] ^= x->s[2]; x->s[0] ^= x->s[3]; x->s[2] ^= t; x->s[3] = rol(x->s[3], 45);
  return r;
}
static uint32_t rank_f64(double m[64][64]) {
  const double eps = 1e-9;
  uint32_t rank = 0;
  int sel[64] = {0};
  for (int i = 0; i < 64; i++) {
    int j = 0;
    while (j < 64 && !(!sel[j] && fabs(m[j][i]) > eps)) j++;
    if (j == 64) continue;
    rank++;
    sel[j] = 1;
    for (int p = i + 1; p < 64; p++) m[j][p] /= m[j][i];
    for (int k = 0; k < 64; k++)
      if (k != j && fabs(m[k][i]) > eps)
        for (int p = i + 1; p < 64; p++) {
          volatile double prod = m[j][p] * m[k][i]; /* two roundings, as Rust: never a fused multiply-subtract */
          m[k][p] -= prod;
        }
  }
  return rank;
}
uint32_t ok_pow_rank_u16(const uint16_t* mat) {
  double m[64][64];
  for (int e = 0; e < 4096; e++) m[e >> 6][e & 63] = (double)mat[e];
  return rank_f64(m);
}
/* Matrix::generate: mat[r][c] nibbles; returns the matrices drawn */
uint32_t ok_pow_generate(const uint8_t seed[32], uint8_t mat[64][64]) {
  xo x;
  for (int i = 0; i < 4; i++) x.s[i] = rd64(seed + 8 * i);
  for (uint32_t tries = 1;; tries++) {
    double m[64][64];
    for (int r = 0; r < 64; r++)
      for (int q = 0; q < 4; q++) {
        uint64_t v = xo_next(&x);
        for (int s = 0; s < 16; s++) mat[r][16 * q + s] = (uint8_t)((v >> (4 * s)) & 15);
      }
    for (int r = 0; r < 64; r++)
      for (int c = 0; c < 64; c++) m[r][c] = mat[r][c];
    if (rank_f64(m) == 64) return tries;
  }
}
void ok_pow_heavy_hash(const uint8_t mat[64][64], const uint8_t in[32], uint8_t out[32]) {
  uint8_t vec[64], prod[32];
  for (int i = 0; i < 32; i++) { vec[2 * i] = in[i] >> 4; vec[2 * i + 1] = in[i] & 15; }
  for (int i = 0; i < 32; i++) {
    uint16_t s1 = 0, s2 = 0;
    for (int j = 0; j < 64; j++) { s1 += mat[2 * i][j] * vec[j]; s2 += mat[2 * i + 1][j] * vec[j]; }
    prod[i] = (uint8_t)(((s1 >> 10) << 4) | (s2 >> 10)) ^ in[i];
  }
  cshake256("HeavyHash", prod, 32, out);
}
static void pow_value(const uint8_t mat[64][64], const uint8_t pre[32], uint64_t timestamp, uint64_t nonce, uint8_t out[32]) {
  uint8_t msg[80], ph[32];
  memset(msg, 0, 80);
  memcpy(msg, pre, 32);
  memcpy(msg + 32, &timestamp, 8);
  memcpy(msg + 72, &nonce, 8);
  cshake256("ProofOfWorkHash", msg, 80, ph);
  ok_pow_heavy_hash(mat, ph, out);
}

/* ---- target, comparison, level ---- */
void ok_pow_compact_target(uint32_t bits, uint8_t out[32]) {
  uint32_t e = bits >> 24, mant, sh;
  if (e <= 3) { mant = (bits & 0xFFFFFF) >> (8 * (3 - e)); sh = 0; }
  else { mant = bits & 0xFFFFFF; sh = 8 * (e - 3); }
  memset(out, 0, 32);
  if (mant > 0x7FFFFF) return;
  sh %= 256;  /* Uint256::overflowing_shl takes the shift modulo 256 */
  for (int k = 0; k < 4; k++) {
    uint32_t bitpos = sh + 8 * k;
    if (bitpos < 256) out[bitpos / 8] = (uint8_t)(mant >> (8 * k));  /* sh is a multiple of 8 */
  }
}
static int le_cmp(const uint8_t a[32], const uint8_t b[32]) {
  for (int i = 31; i >= 0; i--)
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return 0;
}
static uint32_t bits256(const uint8_t a[32]) {
  for (int i = 31; i >= 0; i--)
    if (a[i]) {
      uint32_t b = 0;
      while (a[i] >> b) b++;
      return 8 * i + b;
    }
  return 0;
}

static const uint8_t ORIGIN[32] = {0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe,
                                   0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe, 0xfe};

/* one header: result record, block hash, pow value and pre-PoW hash (any of the three byte outputs may be NULL) */
void ok_pow_validate_one(const ok_header* h, const uint8_t* parents32, const uint32_t* level_len, const ok_header_rules* r, ok_header_result* res,
                         uint8_t* hash32, uint8_t* pow32, uint8_t* pre32) {
  uint8_t pre[32], mat[64][64], pw[32], target[32];
  ok_pow_header_hash(h, parents32, level_len, 0, 0, pre);
  if (hash32) ok_pow_header_hash(h, parents32, level_len, h->nonce, h->timestamp, hash32);
  ok_pow_generate(pre, mat);
  pow_value(mat, pre, h->timestamp, h->nonce, pw);
  ok_pow_compact_target(h->bits, target);
  int genesis = h->n_levels == 0;
  int passed = genesis || le_cmp(pw, target) <= 0;
  int64_t lvl = (int64_t)r->max_block_level - (int64_t)bits256(pw);
  res->level = (uint8_t)(genesis ? r->max_block_level : (lvl > 0 ? lvl : 0));
  res->pow_passed = (uint8_t)passed;
  res->pad_ = 0;
  res->a = res->b = 0;
  uint32_t nd = genesis ? 0 : level_len[h->levels_off];
  const uint8_t* direct = parents32 + 32 * h->parents_off;
  uint64_t max_time = r->now_ms + r->timestamp_deviation_tolerance * 1000;
  res->status = 0;
  if (h->version != r->block_version) { res->status = 1; res->a = h->version; }
  else if (h->timestamp > max_time) { res->status = 2; res->a = h->timestamp; res->b = max_time; }
  else if (nd == 0) res->status = 3;
  else if (nd > r->max_block_parents) { res->status = 4; res->a = nd; res->b = r->max_block_parents; }
  else {
    for (uint32_t k = 0; k < nd && !res->status; k++)
      if (!memcmp(direct + 32 * k, ORIGIN, 32)) res->status = 5;
    if (!res->status && !passed && !(r->flags & 1)) res->status = 6;
  }
  if (pow32) memcpy(pow32, pw, 32);
  if (pre32) memcpy(pre32, pre, 32);
}

typedef struct {
  const ok_header* h;
  const uint8_t* parents32;
  const uint32_t* level_len;
  const ok_header_rules* r;
  ok_header_result* res;
  uint8_t *hash32, *pow32, *pre32;
  size_t lo, hi;
} job;
static void* run_job(void* p) {
  job* j = p;
  for (size_t i = j->lo; i < j->hi; i++)
    ok_pow_validate_one(j->h + i, j->parents32, j->level_len, j->r, j->res + i, j->hash32 ? j->hash32 + 32 * i : NULL,
                        j->pow32 ? j->pow32 + 32 * i : NULL, j->pre32 ? j->pre32 + 32 * i : NULL);
  return NULL;
}
/* n headers over `threads` POSIX threads */
void ok_pow_validate_batch(const ok_header* h, size_t n, const uint8_t* parents32, const uint32_t* level_len, const ok_header_rules* r,
                           ok_header_result* res, uint8_t* hash32, uint8_t* pow32, uint8_t* pre32, int threads) {
  if (threads < 1) threads = 1;
  if (threads > 256) threads = 256;
  pthread_t th[256];
  job jobs[256];
  for (int t = 0; t < threads; t++) {
    jobs[t] = (job){h, parents32, level_len, r, res, hash32, pow32, pre32, n * t / threads, n * (t + 1) / threads};
    pthread_create(&th[t], NULL, run_job, &jobs[t]);
  }
  for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
}

/* the first nonce >= start (at most max_tries of them) whose pow value is <= the header's target: 1 and *nonce_out, or 0 */
int ok_pow_grind(const ok_header* h, const uint8_t* parents32, const uint32_t* level_len, uint64_t start, uint64_t max_tries, uint64_t* nonce_out) {
  uint8_t pre[32], mat[64][64], pw[32], target[32];
  ok_pow_header_hash(h, parents32, level_len, 0, 0, pre);
  ok_pow_generate(pre, mat);
  ok_pow_compact_target(h->bits, target);
  for (uint64_t k = 0; k < max_tries; k++) {
    pow_value(mat, pre, h->timestamp, start + k, pw);
    if (le_cmp(pw, target) <= 0) { *nonce_out = start + k; return 1; }
  }
  return 0;
}
