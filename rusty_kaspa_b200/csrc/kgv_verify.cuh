// kgv_verify.cuh — per-signature verification cores (one signature per thread).
//
// Tri-state verdicts mirror what the reference's script engine can observe
// (crypto/txscript/src/lib.rs:574-643, SURVEY.md §0-7):
//   0 invalid            sig.verify() returned Err            -> Ok(false)
//   1 valid              sig.verify() returned Ok             -> Ok(true)
//   2 pubkey parse error XOnlyPublicKey/PublicKey::from_slice -> Err(InvalidSignature), script aborts
//   3 sig parse error    ecdsa::Signature::from_compact       -> Err(InvalidSignature), script aborts
#pragma once
#include "kgv_secp.cuh"
#include "kgv_sha256.cuh"

namespace kgv {

enum : uint8_t { KGV_ST_INVALID = 0, KGV_ST_VALID = 1, KGV_ST_PK_PARSE = 2, KGV_ST_SIG_PARSE = 3 };

KGV_HD bool fe_words_lt_p(const uint32_t* v) {
  const uint32_t p[8] = {KGV_P0, KGV_P1, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  return lt8(v, p);
}

#define KGV_ST_PENDING 0xFFu  // phase 1 passed: the verdict needs the (batched) inversion of zt

// y^2 = x^3 + 7 for a key given as its tag (2: even y, 3: odd y; a BIP-340 x-only key is tag 2) and the 8 big-endian words of x.
// false: the key does not parse (bad tag, x >= p, or x not on the curve).
KGV_HD bool key_lift(fe& x, fe& y, uint32_t tag, const uint32_t* pkw) {
  if (tag != 2u && tag != 3u) return false;
  limbs_from_be_words(x.v, pkw);
  if (!fe_words_lt_p(x.v)) return false;
  return ge_lift_x(y, x, tag == 3u);
}

// Key record: the part of a verification that depends on the public key alone, prepared once per distinct key of a verify launch
// (k_key_prepare) and copied into the thread's table by every signature under that key.  Words, 16-byte aligned, read with 128-bit loads:
//   [0, 128)   the odd-multiples table {1,3,..,15}*P, entry-major (entry e, word w at 16e + w: x limbs, then y limbs), as build_odd_table leaves it
//   [128, 136) zs, the table's Z scale
//   136        the key's verdict: KGV_ST_VALID (the key parses) or KGV_ST_PK_PARSE; the rest of the record is unset then
#define KGV_KR_ZS 128
#define KGV_KR_STATUS 136
#define KGV_KR_WORDS 140  // 560 bytes
// The comb form's record, for launches whose keys repeat often (key_form, kgv_lib.cu), as k_key_prepare builds it
// (key_joint_record_build) and the verify kernels read it (ecmult_joint).  Words, 64-byte entries, records 64-byte aligned:
//   [0, 16)     P, true affine (x limbs, then y limbs, canonical): ecmult_joint's parity fix
//   16          the key's verdict, as KGV_KR_STATUS; the rest of the record is unset when the key does not parse
//   [32, 2080)  the joint table: entry 32t + 8a + k = (2a+1) * T + (2k-7) * lambda * T, T = 2^(32t) * P, for t = 0..3, a = 0..3,
//               k = 0..7, at word 32 + 16(32t + 8a + k): x limbs, then y limbs, true affine
#define KGV_JR_P 0
#define KGV_JR_STATUS 16
#define KGV_JR_JOINT 32
#define KGV_JR_WORDS (KGV_JR_JOINT + 4 * 32 * 16)  // 2080 words, 8320 bytes
// The host-side reference pair the comb-form record is checked against (the device builds neither record):
// comb key record (key_comb_build; ecmult_comb): four teeth of odd multiples, true affine.  Words, 64-byte entries:
//   [0, 512)   entry 8t + e = (2e+1) * 2^(32t) * P for tooth t = 0..3, e = 0..7, at word 16(8t + e): x limbs, then y limbs
//   512        the key's verdict, as KGV_KR_STATUS
#define KGV_KC_STATUS 512
#define KGV_KC_WORDS 528  // 2112 bytes
// the comb record above, then its joint table (key_joint_build), the same entries as the comb-form record's
//   [528, 2576) entry 32t + 8a + k at word 528 + 16(32t + 8a + k)
#define KGV_KJ_JOINT KGV_KC_WORDS
#define KGV_KJ_WORDS (KGV_KJ_JOINT + 4 * 32 * 16)  // 2576 words, 10304 bytes

// Tab accessor over a key record in global memory (the preparation kernel builds the table in place)
struct RecTab {
  uint32_t* rec;
  KGV_HD void put(int e, int w, uint32_t v) { rec[e * 16 + w] = v; }
  KGV_HD uint32_t get(int e, int w) const { return rec[e * 16 + w]; }
};
// 128-bit read-only load (the records are written by an earlier kernel of the same stream)
KGV_HD void ldg128(uint32_t* w, const uint32_t* p) {
#ifdef __CUDA_ARCH__
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "l"(p));
#else
  for (int i = 0; i < 4; i++) w[i] = p[i];
#endif
}
// a field element at p (16-byte aligned) of a record the same thread writes: two 128-bit accesses (coherent, not the read-only path)
KGV_HD void fe_ld(fe& x, const uint32_t* p) {
#ifdef __CUDA_ARCH__
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
#else
  for (int w = 0; w < 8; w++) x.v[w] = p[w];
#endif
}
KGV_HD void fe_st(uint32_t* p, const fe& x) {
#ifdef __CUDA_ARCH__
  reinterpret_cast<uint4*>(p)[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
#else
  for (int w = 0; w < 8; w++) p[w] = x.v[w];
#endif
}
// table and zs of a prepared key (its verdict is KGV_ST_VALID)
template <class Tab>
KGV_HD void key_rec_load(Tab& tab, fe& zs, const uint32_t* rec) {
#pragma unroll 1
  for (int e = 0; e < 8; e++) {
    uint32_t w[16];
#pragma unroll
    for (int q = 0; q < 4; q++) ldg128(w + 4 * q, rec + 16 * e + 4 * q);
#pragma unroll
    for (int q = 0; q < 16; q++) tab.put(e, q, w[q]);
  }
  ldg128(zs.v, rec + KGV_KR_ZS);
  ldg128(zs.v + 4, rec + KGV_KR_ZS + 4);
}
// fills a key record (tag as for key_lift)
KGV_HD void key_rec_build(uint32_t* rec, uint32_t tag, const uint32_t* pkw) {
  fe x, y, zs;
  uint8_t st = KGV_ST_PK_PARSE;
  if (key_lift(x, y, tag, pkw)) {
    RecTab tab{rec};
    build_odd_table(tab, zs, x, y);
#pragma unroll
    for (int w = 0; w < 8; w++) rec[KGV_KR_ZS + w] = zs.v[w];
    st = KGV_ST_VALID;
  }
  rec[KGV_KR_STATUS] = st;
}
// fills a comb key record: the tooth bases 2^(32t) * P by 96 doublings; each tooth's table as build_odd_table builds one, from the base's
// Jacobian X, Y (affine on the curve with Z scale Z: the table's scale is then zs * Z); one inversion of the four scales' product
// (Montgomery's trick) brings all 32 entries to true affine.
// Host-side reference only (with key_joint_build and ecmult_comb): the device builds key_joint_record_build's record instead.
KGV_HD void key_comb_build(uint32_t* rec, uint32_t tag, const uint32_t* pkw) {
  fe x, y;
  uint8_t st = KGV_ST_PK_PARSE;
  if (key_lift(x, y, tag, pkw)) {
    gej b;
    b.x = x; b.y = y; fe_set_u32(b.z, 1); b.inf = false;
    fe zs[4], pre[4], inv;
#pragma unroll 1
    for (int t = 0; t < 4; t++) {
      if (t) gej_double_n(b, 32);
      RecTab tab{rec + 128 * t};
      fe z;
      build_odd_table(tab, z, b.x, b.y);
      fe_mul(zs[t], z, b.z);
      if (t) fe_mul(pre[t], pre[t - 1], zs[t]);
      else pre[0] = zs[0];
    }
    fe_inv(inv, pre[3]);
#pragma unroll 1
    for (int t = 3; t >= 0; t--) {
      fe zi, zi2, zi3;
      if (t) {
        fe_mul(zi, inv, pre[t - 1]);
        fe_mul(inv, inv, zs[t]);
      } else {
        zi = inv;
      }
      fe_sqr(zi2, zi);
      fe_mul(zi3, zi2, zi);
#pragma unroll 1
      for (int e = 0; e < 8; e++) {
        uint32_t* en = rec + 16 * (8 * t + e);
        fe ex, ey;
        fe_ld(ex, en);
        fe_ld(ey, en + 8);
        fe_mul(ex, ex, zi2);
        fe_mul(ey, ey, zi3);
        fe_st(en, ex);
        fe_st(en + 8, ey);
      }
    }
    st = KGV_ST_VALID;
  }
  rec[KGV_KC_STATUS] = st;
}

// fills the joint table of a comb record whose verdict is KGV_ST_VALID (after key_comb_build).  The host-side reference of
// joint_table_build, which builds the same entries without the comb record.  Per tooth t and pair
// p = (a, j): A = (2a+1) T (comb entry 8t + a) and B = (2j+1) lambda T = (beta x_j, y_j) of comb entry 8t + j; A + B is entry k = j + 4,
// A - B entry k = 3 - j, both affine additions over the one denominator beta x_j - x_A.  The 64 denominators share one inversion
// (Montgomery's trick), with the joint area itself as scratch: beta x_j of tooth t in words 0..7 of entry (t, 0, 3 - j) and the prefix
// product of pairs 0..p (p = 16t + 4a + j) in words 0..7 of entry (t, a, j + 4), each read before the pass going back down overwrites it.
// No denominator is zero for a key that parses: A = +-B means (2a+1) = +-(2j+1) lambda (mod n), so (2a+1)^3 = +-(2j+1)^3 (mod n) with
// both cubes below 7^3 < n, hence 2a+1 = 2j+1 as integers and lambda = +-1, which it is not.
// About 860 products: 16 by beta, 63 + 126 for the trick, 6 per pair, one fe_inv.
// Each thread owns a 10 KB record, so a warp's accesses are 32 lanes at a 10 KB stride: all of them go through fe_ld / fe_st (128-bit),
// and every operand is loaded once per loop level that needs it.
KGV_HD void key_joint_build(uint32_t* rec) {
  const fe beta = {KGV_BETA_LIMBS};
  uint32_t* jt = rec + KGV_KJ_JOINT;
#pragma unroll 1
  for (int t = 0; t < 4; t++) {
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
      fe bx;
      fe_ld(bx, rec + 16 * (8 * t + j));
      fe_mul(bx, bx, beta);
      fe_st(jt + 16 * (32 * t + 3 - j), bx);
    }
  }
  fe acc;
  fe_set_u32(acc, 1);
#pragma unroll 1
  for (int ta = 0; ta < 16; ta++) {  // pairs p = 4 ta + j
    const int t = ta >> 2, a = ta & 3;
    fe xa;
    fe_ld(xa, rec + 16 * (8 * t + a));
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
      fe bx, d;
      fe_ld(bx, jt + 16 * (32 * t + 3 - j));
      fe_sub(d, bx, xa);
      fe_mul(acc, acc, d);
      fe_st(jt + 16 * (32 * t + 8 * a + j + 4), acc);
    }
  }
  fe inv;
  fe_inv(inv, acc);
#pragma unroll 1
  for (int ta = 15; ta >= 0; ta--) {
    const int t = ta >> 2, a = ta & 3;
    fe xa, ya;
    fe_ld(xa, rec + 16 * (8 * t + a));
    fe_ld(ya, rec + 16 * (8 * t + a) + 8);
#pragma unroll 1
    for (int j = 3; j >= 0; j--) {
      const int p = 4 * ta + j, q = p - 1;
      fe bx, yb, d, di;
      fe_ld(bx, jt + 16 * (32 * t + 3 - j));
      fe_ld(yb, rec + 16 * (8 * t + j) + 8);
      if (p) {
        fe pre;
        fe_ld(pre, jt + 16 * (32 * (q >> 4) + 8 * ((q >> 2) & 3) + (q & 3) + 4));
        fe_sub(d, bx, xa);
        fe_mul(di, inv, pre);
        fe_mul(inv, inv, d);
      } else {
        di = inv;
      }
#pragma unroll 1
      for (int sgn = 0; sgn < 2; sgn++) {  // A + B (k = j + 4), then A - B (k = 3 - j)
        fe l, x3, y3, t1;
        if (sgn) fe_neg(t1, yb);
        else t1 = yb;
        fe_sub(t1, t1, ya);
        fe_mul(l, t1, di);                 // slope
        fe_sqr(x3, l);
        fe_sub(x3, x3, xa);
        fe_sub(x3, x3, bx);                // x3 = l^2 - xA - xB
        fe_sub(t1, xa, x3);
        fe_mul(y3, l, t1);
        fe_sub(y3, y3, ya);                // y3 = l (xA - x3) - yA
        uint32_t* en = jt + 16 * (32 * t + 8 * a + (sgn ? 3 - j : j + 4));
        fe_st(en, x3);
        fe_st(en + 8, y3);
      }
    }
  }
}

// build_odd_table's Tab over four entries of local field-element arrays (x limbs in x[e], y limbs in y[e])
struct FeTab {
  fe* x;
  fe* y;
  KGV_HD void put(int e, int w, uint32_t v) {
    if (w < 8) x[e].v[w] = v;
    else y[e].v[w - 8] = v;
  }
  KGV_HD uint32_t get(int e, int w) const { return w < 8 ? x[e].v[w] : y[e].v[w - 8]; }
};
// fills the joint table jt (KGV_JR_JOINT's layout) of the key P = (px, py), affine.  It builds only the tooth entries the table is made
// of, A = (2a+1) T_t and B = (2j+1) lambda T_t for a, j < 4, and runs one inversion:
//  1. per tooth: the base T_t = 2^(32t) P by 32 doublings, then {1,3,5,7} T_t by build_odd_table<4> in the tooth's frame: entry e is
//     (X'_e, Y'_e) = (x_e Z_t^2, y_e Z_t^3), Z_t the table's scale times the base's Z; and beta X'_e.
//  2. one Montgomery trick over the 64 frame denominators d'_p = beta X'_j - X'_a (pair p = 16t + 4a + j) and then the four Z_t;
//     one fe_inv.
//  3. going back down, the Z_t's inverses bring the 16 tooth entries and their beta X to true affine, in place (3 products each), then
//     per pair 1 / (beta x_j - x_a) = Z_t^2 / d'_p (one product) and A + B (entry k = j + 4), A - B (k = 3 - j) as key_joint_build
//     forms them (6 products).
// No d'_p is zero (key_joint_build's argument; Z_t != 0).
// All scratch (tooth entries, denominators, prefix products: 5.9 KB) is in local arrays, which the hardware interleaves across a warp's
// lanes: a warp's access to one element is coalesced.  The record itself is 8 KB per thread, so a warp's access to it touches 32 sectors
// at an 8 KB stride; only the 256 16-byte stores of the finished entries go there (with the scratch in the record, k_key_prepare took
// 2.54 ms at the bench shape, 2.24 ms with it in local arrays; DESIGN.md §4 K1).
// About 1 000 products: 16 by beta, 67 + 4 * 5 + 126 for the trick, 48 to true affine, 7 per pair (448), one fe_inv.
KGV_HD void joint_table_build(uint32_t* jt, const fe& px, const fe& py) {
  const fe beta = {KGV_BETA_LIMBS};
  fe ex[16], ey[16], eb[16];  // tooth t, entry e at 4t + e: x, y, beta x (in the frame, then true affine)
  fe dn[64], pre[64];         // d'_p and the prefix product of d'_0..d'_p
  fe zs[4], zp[5];            // Z_t; zp[t]: the prefix product of the 64 denominators and Z_0..Z_{t-1}
  gej b;
  b.x = px; b.y = py; fe_set_u32(b.z, 1); b.inf = false;
#pragma unroll 1
  for (int t = 0; t < 4; t++) {
    if (t) gej_double_n(b, 32);
    FeTab tab{ex + 4 * t, ey + 4 * t};
    fe z;
    build_odd_table<4>(tab, z, b.x, b.y);
    fe_mul(zs[t], z, b.z);
#pragma unroll 1
    for (int e = 0; e < 4; e++) fe_mul(eb[4 * t + e], ex[4 * t + e], beta);
  }
  fe acc;
#pragma unroll 1
  for (int p = 0; p < 64; p++) {
    const int t = p >> 4, a = (p >> 2) & 3, j = p & 3;
    fe d;
    fe_sub(d, eb[4 * t + j], ex[4 * t + a]);
    if (p) fe_mul(acc, acc, d);
    else acc = d;
    dn[p] = d;
    pre[p] = acc;
  }
  zp[0] = acc;
#pragma unroll 1
  for (int t = 0; t < 4; t++) {
    fe_mul(acc, acc, zs[t]);
    zp[t + 1] = acc;
  }
  fe inv;
  fe_inv(inv, acc);
#pragma unroll 1
  for (int t = 3; t >= 0; t--) {
    fe zi, zi2, zi3;
    fe_mul(zi, inv, zp[t]);
    fe_mul(inv, inv, zs[t]);
    fe_sqr(zi2, zi);
    fe_mul(zi3, zi2, zi);
    fe_sqr(zs[t], zs[t]);  // Z_t^2 from here on
#pragma unroll 1
    for (int e = 4 * t; e < 4 * t + 4; e++) {
      fe_mul(ex[e], ex[e], zi2);
      fe_mul(ey[e], ey[e], zi3);
      fe_mul(eb[e], eb[e], zi2);
    }
  }
  // inv = 1 / (d'_0 ... d'_63)
#pragma unroll 1
  for (int p = 63; p >= 0; p--) {
    const int t = p >> 4, a = (p >> 2) & 3, j = p & 3;
    fe di;
    if (p) {
      fe_mul(di, inv, pre[p - 1]);
      fe_mul(inv, inv, dn[p]);
    } else {
      di = inv;
    }
    fe_mul(di, di, zs[t]);  // 1 / (beta x_j - x_a)
    const fe xa = ex[4 * t + a], ya = ey[4 * t + a], bx = eb[4 * t + j], yb = ey[4 * t + j];
#pragma unroll 1
    for (int sgn = 0; sgn < 2; sgn++) {  // A + B (k = j + 4), then A - B (k = 3 - j)
      fe l, x3, y3, t1;
      if (sgn) fe_neg(t1, yb);
      else t1 = yb;
      fe_sub(t1, t1, ya);
      fe_mul(l, t1, di);                 // slope
      fe_sqr(x3, l);
      fe_sub(x3, x3, xa);
      fe_sub(x3, x3, bx);                // x3 = l^2 - xA - xB
      fe_sub(t1, xa, x3);
      fe_mul(y3, l, t1);
      fe_sub(y3, y3, ya);                // y3 = l (xA - x3) - yA
      uint32_t* en = jt + 16 * (32 * t + 8 * a + (sgn ? 3 - j : j + 4));
      fe_st(en, x3);
      fe_st(en + 8, y3);
    }
  }
}
// fills a comb-form record (KGV_JR_*; tag as for key_lift)
KGV_HD void key_joint_record_build(uint32_t* rec, uint32_t tag, const uint32_t* pkw) {
  fe x, y;
  uint8_t st = KGV_ST_PK_PARSE;
  if (key_lift(x, y, tag, pkw)) {
    fe_st(rec + KGV_JR_P, x);
    fe_st(rec + KGV_JR_P + 8, y);
    joint_table_build(rec + KGV_JR_JOINT, x, y);
    st = KGV_ST_VALID;
  }
  rec[KGV_JR_STATUS] = st;
}

// Where the key part of a verification comes from: the key's comb record (comb), its plain record, or none (rec == nullptr: the key is
// lifted and its odd-multiples table built per signature).
struct KeySrc {
  const uint32_t* rec;
  bool comb;
};
// a prepared key's verdict: false when the key does not parse
KGV_HD bool key_rec_valid(const KeySrc& key) { return key.rec[key.comb ? KGV_JR_STATUS : KGV_KR_STATUS] == KGV_ST_VALID; }
// R = kP*P + kG*G and zt, the true Z of R (unset when R is infinity).  px, py: the key, read on the inline path only.
template <class Tab, class GLoad, class Trace = NoTrace>
KGV_HD void ecmult_key(gej& R, fe& zt, const KeySrc& key, const fe& px, const fe& py, const uint32_t* kP, const uint32_t* kG, Tab& tab,
                       const uint32_t* gtab, GLoad gload, Trace trace = Trace()) {
  fe zs;
  if (key.comb) {
    ecmult_joint(R, kP, kG, key.rec + KGV_JR_P, key.rec + KGV_JR_JOINT, tab, gtab, gload);
  } else {
    if (key.rec) key_rec_load(tab, zs, key.rec);
    else build_odd_table(tab, zs, px, py);
    ecmult_double(R, zs, kP, kG, tab, gtab, gload, trace);
  }
  if (R.inf) return;
  if (key.comb) zt = R.z;  // comb entries are true affine
  else fe_mul(zt, R.z, zs);
}

// BIP-340 verification, phase 1: everything up to the projective result R = s*G - e*P.
// pkw/mw: 8 big-endian words, sigw: 16 big-endian words (r || s).  Returns a final verdict, or KGV_ST_PENDING with (X, Y, zt = true Z, rx)
// filled in.
template <class Tab, class GLoad, class Trace = NoTrace>
KGV_HD uint8_t schnorr_phase1(fe& X, fe& Y, fe& zt, fe& rx, const uint32_t* pkw, const uint32_t* mw, const uint32_t* sigw, Tab& tab,
                              const uint32_t* gtab, GLoad gload, const KeySrc& key, Trace trace = Trace()) {
  fe px, py;
  if (key.rec) {
    if (!key_rec_valid(key)) return KGV_ST_PK_PARSE;
  } else {
    limbs_from_be_words(px.v, pkw);
    if (!fe_words_lt_p(px.v)) return KGV_ST_PK_PARSE;      // x >= p
    trace(1, px.v, 8);
    if (!ge_lift_x(py, px, false)) return KGV_ST_PK_PARSE;  // not on the curve
    trace(2, py.v, 8);
  }
  limbs_from_be_words(rx.v, sigw);
  if (!fe_words_lt_p(rx.v)) return KGV_ST_INVALID;        // r >= p
  uint32_t s[8], e[8], k[8], ew[8];
  limbs_from_be_words(s, sigw + 8);
  if (sc_ge_n(s)) return KGV_ST_INVALID;                  // s >= n
  bip340_challenge(ew, sigw, pkw, mw);
#pragma unroll
  for (int i = 0; i < 8; i++) e[7 - i] = ew[i];
  sc_reduce_once(e);
  sc_neg(k, e);                                           // R = s*G - e*P
  trace(3, e, 8); trace(4, k, 8); trace(5, s, 8);
  gej R;
  ecmult_key(R, zt, key, px, py, k, s, tab, gtab, gload, trace);
  { uint32_t f[1] = {R.inf}; trace(18, f, 1); }
  if (R.inf) return KGV_ST_INVALID;
  trace(19, R.x.v, 8); trace(20, R.y.v, 8); trace(21, R.z.v, 8);
  X = R.x;
  Y = R.y;
  return KGV_ST_PENDING;
}
// phase 2: zi = 1/zt. Valid iff y(R) is even and x(R) == r.
template <class Trace = NoTrace>
KGV_HD uint8_t schnorr_phase2(const fe& X, const fe& Y, const fe& zi, const fe& rx, Trace trace = Trace()) {
  fe zi2, ax, ay;
  fe_sqr(zi2, zi);
  fe_mul(ax, X, zi2);
  fe_mul(ay, Y, zi2);
  fe_mul(ay, ay, zi);
  fe_normalize(ay);
  fe_normalize(ax);
  trace(22, ax.v, 8); trace(23, ay.v, 8);
  if (ay.v[0] & 1u) return KGV_ST_INVALID;                // y(R) odd
  bool eq = true;
#pragma unroll
  for (int i = 0; i < 8; i++) eq = eq && (ax.v[i] == rx.v[i]);
  return eq ? KGV_ST_VALID : KGV_ST_INVALID;
}
// single-signature form (audit kernel, host unit tests)
template <class Tab, class GLoad, class Trace = NoTrace>
KGV_HD uint8_t schnorr_verify_core(const uint32_t* pkw, const uint32_t* mw, const uint32_t* sigw, Tab& tab, const uint32_t* gtab,
                                   GLoad gload, Trace trace = Trace(), KeySrc key = KeySrc{nullptr, false}) {
  fe X, Y, zt, rx, zi;
  uint8_t st = schnorr_phase1(X, Y, zt, rx, pkw, mw, sigw, tab, gtab, gload, key, trace);
  if (st != KGV_ST_PENDING) return st;
  fe_inv(zi, zt);
  return schnorr_phase2(X, Y, zi, rx, trace);
}

// ECDSA verification with libsecp256k1 semantics, phase 1: parsing and range checks.
// pkw: 8 big-endian words of x, tag = first key byte.  Returns a final verdict or KGV_ST_PENDING with the key (qx,qy; unset with a record),
// r, s (to be inverted, possibly batched) and the reduced message m.
KGV_HD uint8_t ecdsa_phase1(fe& qx, fe& qy, uint32_t* r, uint32_t* s, uint32_t* m, uint32_t tag, const uint32_t* pkw, const uint32_t* mw,
                            const uint32_t* sigw, const KeySrc& key) {
  if (key.rec) {
    if (!key_rec_valid(key)) return KGV_ST_PK_PARSE;
  } else if (!key_lift(qx, qy, tag, pkw)) {
    return KGV_ST_PK_PARSE;
  }
  limbs_from_be_words(r, sigw);
  limbs_from_be_words(s, sigw + 8);
  if (sc_ge_n(r) || sc_ge_n(s)) return KGV_ST_SIG_PARSE;  // from_compact rejects overflow
  limbs_from_be_words(m, mw);
  sc_reduce_once(m);
  if (sc_is_high(s)) return KGV_ST_INVALID;               // verify requires low S
  if (is_zero8(r) || is_zero8(s)) return KGV_ST_INVALID;
  return KGV_ST_PENDING;
}
// phase 2: sn = s^-1 mod n.  R = (m/s)*G + (r/s)*Q, valid iff x(R) mod n == r.
template <class Tab, class GLoad>
KGV_HD uint8_t ecdsa_phase2(const fe& qx, const fe& qy, const uint32_t* r, const uint32_t* sn, const uint32_t* m, Tab& tab, const uint32_t* gtab,
                            GLoad gload, const KeySrc& key) {
  uint32_t u1[8], u2[8];
  sc_mul(u1, sn, m);
  sc_mul(u2, sn, r);
  gej R;
  fe zt;
  ecmult_key(R, zt, key, qx, qy, u2, u1, tab, gtab, gload);
  if (R.inf) return KGV_ST_INVALID;
  // x(R) mod n == r  <=>  X == r*Zt^2  or  (r + n < p and X == (r+n)*Zt^2)
  fe zt2, t, rf;
  fe_sqr(zt2, zt);
#pragma unroll
  for (int i = 0; i < 8; i++) rf.v[i] = r[i];
  fe_mul(t, rf, zt2);
  if (fe_equal(t, R.x)) return KGV_ST_VALID;
  const uint32_t n[8] = KGV_N_LIMBS;
  uint32_t rn[8];
  uint32_t c = add8(rn, r, n);
  if (c || !fe_words_lt_p(rn)) return KGV_ST_INVALID;     // r + n >= p
#pragma unroll
  for (int i = 0; i < 8; i++) rf.v[i] = rn[i];
  fe_mul(t, rf, zt2);
  return fe_equal(t, R.x) ? KGV_ST_VALID : KGV_ST_INVALID;
}
template <class Tab, class GLoad>
KGV_HD uint8_t ecdsa_verify_core(uint32_t tag, const uint32_t* pkw, const uint32_t* mw, const uint32_t* sigw, Tab& tab,
                                 const uint32_t* gtab, GLoad gload, KeySrc key = KeySrc{nullptr, false}) {
  fe qx, qy;
  uint32_t r[8], s[8], m[8], sn[8];
  uint8_t st = ecdsa_phase1(qx, qy, r, s, m, tag, pkw, mw, sigw, key);
  if (st != KGV_ST_PENDING) return st;
  sc_inv(sn, s);
  return ecdsa_phase2(qx, qy, r, sn, m, tab, gtab, gload, key);
}

// One entry of the generator tables: v * B for v in [1, 65535], B affine; result affine.
KGV_HD void gtab_entry(fe& ox, fe& oy, uint32_t v, const fe& bx, const fe& by) {
  gej r;
  r.inf = true;
  fe_set_zero(r.x); fe_set_zero(r.y); fe_set_zero(r.z);
  for (int bit = 15; bit >= 0; bit--) {
    gej_double(r);
    if ((v >> bit) & 1u) gej_add_ge(r, bx, by);
  }
  fe zi, zi2;
  fe_inv(zi, r.z);
  fe_sqr(zi2, zi);
  fe_mul(ox, r.x, zi2);
  fe_mul(oy, r.y, zi2);
  fe_mul(oy, oy, zi);
  fe_normalize(ox);
  fe_normalize(oy);
}

#define KGV_GX_LIMBS {0x16F81798u, 0x59F2815Bu, 0x2DCE28D9u, 0x029BFCDBu, 0xCE870B07u, 0x55A06295u, 0xF9DCBBACu, 0x79BE667Eu}
#define KGV_GY_LIMBS {0xFB10D4B8u, 0x9C47D08Fu, 0xA6855419u, 0xFD17B448u, 0x0E1108A8u, 0x5DA4FBFCu, 0x26A3C465u, 0x483ADA77u}
// 2^128 * G (tools/derive_constants.py)
#define KGV_G128X_LIMBS {0x9EC4C0DAu, 0x1B7B444Cu, 0x723EA335u, 0xE88C5678u, 0x981F162Eu, 0x9239C1ADu, 0xF63B5F33u, 0x8F68B9D2u}
#define KGV_G128Y_LIMBS {0x501FFF82u, 0xF23CBF79u, 0x95510BFDu, 0xBBEA2CFEu, 0xB6BE215Du, 0xDE1D90C2u, 0xBA063986u, 0x662A9F2Du}
// 2^(32j) * G for the other generator tables (oracle/pyref.py: pt_mul(2**(32*j), G); tests/test_hostsim_comb.py checks them)
#define KGV_G32X_LIMBS {0x39A48DB0u, 0xEFD7835Bu, 0x9B3C03BFu, 0x9F1215A2u, 0x9B7BDE45u, 0x2791D0A0u, 0x696E7167u, 0x100F44DAu}
#define KGV_G32Y_LIMBS {0x2BC65A09u, 0x0FBD5CD6u, 0xFF5195ACu, 0xB7FF4A18u, 0x0C090666u, 0x2EC8F330u, 0x92A00B77u, 0xCDD9E131u}
#define KGV_G64X_LIMBS {0x42D0E6BDu, 0x13B7E0E7u, 0xDB0F5E53u, 0xF774D163u, 0x104D6ECBu, 0x82A2147Cu, 0x243C4E25u, 0x3322D401u}
#define KGV_G64Y_LIMBS {0x6C28B2A0u, 0x24F3A2E9u, 0xA2873AF6u, 0x2805F63Eu, 0x4DDAF9B7u, 0xBFB019BCu, 0xE9664EF5u, 0x56E70797u}
#define KGV_G96X_LIMBS {0x40FB27B6u, 0x32427E28u, 0xBE430576u, 0xC76E3DB2u, 0x61686AA5u, 0x10F238ADu, 0xBE778B1Bu, 0xFEA74E3Du}
#define KGV_G96Y_LIMBS {0xF23CB96Fu, 0x701D3DB7u, 0x973F7B77u, 0x126B596Bu, 0xCCB6AF93u, 0x7CF674DEu, 0x9B0B1329u, 0x6E0568DBu}
#define KGV_G160X_LIMBS {0xAC1F98CDu, 0xCBFC99C8u, 0x4D7F0308u, 0x52348905u, 0x1CC66021u, 0xFAED8A9Cu, 0x4A474870u, 0x9C3919A8u}
#define KGV_G160Y_LIMBS {0xD4FC599Du, 0xBE7E5E03u, 0x6C64C8E6u, 0x905326F7u, 0xF260E641u, 0x584F044Bu, 0x4A4DDD57u, 0xDDB84F0Fu}
#define KGV_G192X_LIMBS {0x2120E2B3u, 0x7F3B58FAu, 0x7F47F9AAu, 0x7A58FDCEu, 0x4CE6E521u, 0xE7BE4AE3u, 0x1F51BDBAu, 0xEAA649F2u}
#define KGV_G192Y_LIMBS {0xBA5AD93Du, 0xD47A5305u, 0xF13F7E59u, 0x01A6B965u, 0x9879AA5Au, 0xC69A80F8u, 0x5BBBB03Au, 0xBE3279EDu}
#define KGV_G224X_LIMBS {0x9475B7BAu, 0x884FDFF0u, 0xE4918B3Du, 0xE039E730u, 0xF5018CDBu, 0x3D3E57EDu, 0x1943785Cu, 0x95939698u}
#define KGV_G224Y_LIMBS {0x7524F2FDu, 0xE9B8ABF8u, 0xC8709385u, 0x9C653F64u, 0x4B9CD684u, 0x8BA0386Au, 0x88C331DDu, 0x2E7E5528u}
// base of generator table j (0..7): 2^(32j) * G
KGV_HD void gtab_base(fe& x, fe& y, int j) {
  const fe bx[8] = {{KGV_GX_LIMBS}, {KGV_G32X_LIMBS}, {KGV_G64X_LIMBS}, {KGV_G96X_LIMBS}, {KGV_G128X_LIMBS}, {KGV_G160X_LIMBS}, {KGV_G192X_LIMBS}, {KGV_G224X_LIMBS}};
  const fe by[8] = {{KGV_GY_LIMBS}, {KGV_G32Y_LIMBS}, {KGV_G64Y_LIMBS}, {KGV_G96Y_LIMBS}, {KGV_G128Y_LIMBS}, {KGV_G160Y_LIMBS}, {KGV_G192Y_LIMBS}, {KGV_G224Y_LIMBS}};
  x = bx[j];
  y = by[j];
}

}  // namespace kgv
