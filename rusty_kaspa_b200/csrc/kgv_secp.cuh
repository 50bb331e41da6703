// kgv_secp.cuh — secp256k1 group law, GLV split, window recoding and the double-scalar
// multiplication R = kP*P + kG*G used by both verifiers (BIP-340 Schnorr, ECDSA).
//
// GPU-native restructuring of what libsecp256k1's ecmult does for the reference
// (crypto/txscript/src/lib.rs:593, :628):
//   * one signature per thread, branch-uniform fixed windows (no wNAF: no per-lane divergence)
//   * P part: GLV split kP = k1 + k2*lambda (|k1|,|k2| < 2^128), signed odd 4-bit digits
//     (33 digits each, never zero), 8-entry table {1,3,..,15}*P per thread in shared memory,
//     built on an isomorphic curve so the entries are affine ("effective affine")
//   * G part: kG = lo + 2^128*hi, unsigned 16-bit windows into two 65536-entry affine tables
//     (G and 2^128*G of the eight 2^(32j)*G tables, L2 resident), 16 mixed additions
//   * 128 shared doublings
// ecmult_comb is the same product for a key prepared once per launch as a four-tooth comb (keys that repeat often): 32 doublings.
// ecmult_joint (the device's ladder for such keys) reads joint entries a*T + b*lambda*T of the same teeth: one addition per digit pair of
// both GLV halves, 44 instead of 66, and 30 doublings.  ecmult_comb stays as the host-checked reference it is compared with.
#pragma once
#include "kgv_arith.cuh"

namespace kgv {

// ------------------------------------------------------------------------------------------
// constants
// ------------------------------------------------------------------------------------------
// group order n, little-endian limbs
#define KGV_N_LIMBS {0xD0364141u, 0xBFD25E8Cu, 0xAF48A03Bu, 0xBAAEDCE6u, 0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}
// beta: cube root of unity mod p with lambda*(x,y) = (beta*x, y)
#define KGV_BETA_LIMBS {0x719501EEu, 0xC1396C28u, 0x12F58995u, 0x9CF04975u, 0xAC3434E9u, 0x6E64479Eu, 0x657C0710u, 0x7AE96A2Bu}
// GLV lattice (derived in tools/derive_constants.py): g1 = round(2^384*b2/n), g2 = round(2^384*(-b1)/n)
#define KGV_G1_LIMBS {0x45DBB031u, 0xE893209Au, 0x71E8CA7Fu, 0x3DAA8A14u, 0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u}
#define KGV_G2_LIMBS {0x8AC47F71u, 0x1571B4AEu, 0x9DF506C6u, 0x221208ACu, 0x0ABFE4C4u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u}
// a1 = b2 (126 bits), |b1| (128 bits), a2 (129 bits) as 5 limbs
#define KGV_A1_LIMBS {0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u, 0u}
#define KGV_MB1_LIMBS {0x0ABFE4C3u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u, 0u}
#define KGV_A2_LIMBS {0x9D44CFD8u, 0x57C1108Du, 0xA8E2F3F6u, 0x14CA50F7u, 1u}

struct gej {
  fe x, y, z;
  bool inf;
};

// Optional intermediate-value tracing (audit/debug kernels and the host unit tests use it to
// compare device and host executions stage by stage); NoTrace compiles to nothing.
struct NoTrace {
  KGV_HD void operator()(int /*stage*/, const uint32_t* /*words*/, int /*n*/) const {}
};

// ------------------------------------------------------------------------------------------
// scalars (mod n): only what verification needs
// ------------------------------------------------------------------------------------------
// a >= n ?
KGV_HD bool sc_ge_n(const uint32_t* a) {
  const uint32_t n[8] = KGV_N_LIMBS;
  return !lt8(a, n);
}
// a in [0, 2^256) -> a mod n (2^256 < 2n: one conditional subtraction)
KGV_HD void sc_reduce_once(uint32_t* a) {
  const uint32_t n[8] = KGV_N_LIMBS;
  uint32_t t[8];
  uint32_t bo = sub8(t, a, n);
  if (!bo) {
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = t[i];
  }
}
KGV_HD bool is_zero8(const uint32_t* a) { return (a[0] | a[1] | a[2] | a[3] | a[4] | a[5] | a[6] | a[7]) == 0; }
// r = -a mod n, for a in [0,n)
KGV_HD void sc_neg(uint32_t* r, const uint32_t* a) {
  const uint32_t n[8] = KGV_N_LIMBS;
  if (is_zero8(a)) {
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = 0;
    return;
  }
  (void)sub8(r, n, a);
}

// ---- full scalar multiplication / inversion mod n (ECDSA only) ----
// acc[0..NA) += x[0..NX) * (2^256 - n); carries propagate to the top limb
template <int NA, int NX>
KGV_HD void sc_fold(uint32_t* acc, const uint32_t* x) {
  const uint32_t nc[5] = {0x2FC9BEBFu, 0x402DA173u, 0x50B75FC4u, 0x45512319u, 1u};
#pragma unroll
  for (int i = 0; i < NX; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 5; j++) {
      if (i + j < NA) {
        uint64_t t = (uint64_t)x[i] * nc[j] + acc[i + j] + c;
        acc[i + j] = (uint32_t)t;
        c = t >> 32;
      }
    }
#pragma unroll
    for (int k = i + 5; k < NA; k++) {
      c += acc[k];
      acc[k] = (uint32_t)c;
      c >>= 32;
    }
  }
}
// r = t mod n for a 512-bit t
KGV_HD void sc_reduce512(uint32_t* r, const uint32_t* t) {
  uint32_t a[13], b[9], c[9];
#pragma unroll
  for (int i = 0; i < 13; i++) a[i] = i < 8 ? t[i] : 0u;
  sc_fold<13, 8>(a, t + 8);          // < 2^386
#pragma unroll
  for (int i = 0; i < 9; i++) b[i] = i < 8 ? a[i] : 0u;
  sc_fold<9, 5>(b, a + 8);           // < 2^260
#pragma unroll
  for (int i = 0; i < 9; i++) c[i] = i < 8 ? b[i] : 0u;
  sc_fold<9, 1>(c, b + 8);           // < 2^256 + 2^133
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = c[i];
  uint32_t top = c[8];               // 0 or 1; if 1 the low part is tiny
  {
    uint32_t one[1] = {top};
    uint32_t d[8];
#pragma unroll
    for (int i = 0; i < 8; i++) d[i] = r[i];
    sc_fold<8, 1>(d, one);
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = d[i];
  }
  sc_reduce_once(r);
}
// As for fe_mul / fe_sqr, the device versions are real functions (operands by value, in registers): ALL scalar arithmetic of the ECDSA
// kernel goes through ONE non-inlined function, r = a^(2^k) * (b or 1), with a single copy of the 8x8 product and of the reduction (squarings
// use the general product: +28 multiplies each, 0.4 % more instructions per verification).  Three separate blocks (multiply, square,
// run-of-squarings: ~19 KB of SASS next to the 25 KB of the point arithmetic) pushed the kernel's hot code out of the instruction cache: ncu
// showed `no_instruction` stalls at 1.88 per issued instruction against 0.75 in the Schnorr kernel.  The host unit-test build inlines them.
#if defined(__CUDACC__)
struct sc8 { uint32_t v[8]; };
static __device__ __noinline__ sc8 sc_pow2k_mul_call(sc8 a, int k, int with_mul, sc8 b) {
  const int n = k + with_mul;
#pragma unroll 1
  for (int i = 0; i < n; i++) {
    sc8 y;
#pragma unroll
    for (int w = 0; w < 8; w++) y.v[w] = i < k ? a.v[w] : b.v[w];
    uint32_t t[16];
    mul_wide(t, a.v, y.v);
    sc_reduce512(a.v, t);
  }
  return a;
}
KGV_HD void sc_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  sc8 x, y;
#pragma unroll
  for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  sc8 z = sc_pow2k_mul_call(x, 0, 1, y);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}
KGV_HD void sc_sqr(uint32_t* r, const uint32_t* a) {
  sc8 x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = a[i];
  sc8 z = sc_pow2k_mul_call(x, 1, 0, x);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}
// r = r^(2^k) * m
KGV_HD void sc_sqr_n_mul(uint32_t* r, int k, const uint32_t* m) {
  sc8 x, y;
#pragma unroll
  for (int i = 0; i < 8; i++) { x.v[i] = r[i]; y.v[i] = m[i]; }
  sc8 z = sc_pow2k_mul_call(x, k, 1, y);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
}
#else
KGV_HD void sc_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t t[16];
  mul_wide(t, a, b);
  sc_reduce512(r, t);
}
KGV_HD void sc_sqr(uint32_t* r, const uint32_t* a) {
  uint32_t t[16];
  sqr_wide(t, a);
  sc_reduce512(r, t);
}
KGV_HD void sc_sqr_n(uint32_t* r, int n) {
  for (int i = 0; i < n; i++) sc_sqr(r, r);
}
// r = r^(2^k) * m
KGV_HD void sc_sqr_n_mul(uint32_t* r, int k, const uint32_t* m) { sc_sqr_n(r, k); sc_mul(r, r, m); }
#endif
// r = a^(n-2) mod n (a != 0).  The exponent is public and identical in every lane: no divergence.  Addition chain: the 127 leading one bits
// of n-2 through x_k = a^(2^k - 1) (k = 2, 3, 6, 8, 14, 28, 56, 112, 126: the ladder libsecp256k1's scalar inverse uses), the remaining 129 bits
// by a sliding window over the odd powers a, a^3, a^5, a^7 (schedule derived and checked against pow(a, n-2, n) by
// tools/derive_sc_inv_chain.py; tests/test_hostsim.py runs this very function on the host): 255 squarings + 44 multiplications instead of the 255 + 191
// of plain square-and-multiply (ECDSA shares one inversion among KGV_ITEMS signatures; it was 11 % of an ECDSA verification).
KGV_HD void sc_inv(uint32_t* r, const uint32_t* a) {
  uint32_t a1[8], a3[8], a5[8], a7[8], x6[8], x14[8], t[8], u[8];
#pragma unroll
  for (int i = 0; i < 8; i++) a1[i] = a[i];
  sc_sqr(u, a1);                       // a^2
  sc_mul(a3, u, a1);                   // x2 = a^3
  sc_mul(a5, a3, u);                   // a^5
  sc_sqr(t, a3); sc_mul(a7, t, a1);    // x3 = a^7
#pragma unroll
  for (int i = 0; i < 8; i++) t[i] = a7[i];
  sc_sqr_n_mul(t, 3, a7);                                              // x6
#pragma unroll
  for (int i = 0; i < 8; i++) x6[i] = t[i];
  sc_sqr_n_mul(t, 2, a3);                                              // x8
  sc_sqr_n_mul(t, 6, x6);                                              // x14
#pragma unroll
  for (int i = 0; i < 8; i++) x14[i] = t[i];
  sc_sqr_n_mul(t, 14, x14);                                            // x28
#pragma unroll
  for (int i = 0; i < 8; i++) u[i] = t[i];
  sc_sqr_n_mul(t, 28, u);                                              // x56
#pragma unroll
  for (int i = 0; i < 8; i++) u[i] = t[i];
  sc_sqr_n_mul(t, 56, u);                                              // x112
  sc_sqr_n_mul(t, 14, x14);                                            // x126
  sc_sqr_n_mul(t, 1, a1);                                              // the 127 leading ones
#define SC_STEP(k, x) sc_sqr_n_mul(t, k, x);
  SC_STEP(4, a5) SC_STEP(2, a3) SC_STEP(4, a5) SC_STEP(4, a5) SC_STEP(2, a3) SC_STEP(3, a3)
  SC_STEP(4, a7) SC_STEP(5, a7) SC_STEP(4, a3) SC_STEP(4, a5) SC_STEP(4, a7) SC_STEP(3, a5)
  SC_STEP(3, a1) SC_STEP(6, a5) SC_STEP(10, a7) SC_STEP(4, a7) SC_STEP(4, a7) SC_STEP(3, a7)
  SC_STEP(2, a3) SC_STEP(2, a1) SC_STEP(3, a1) SC_STEP(5, a5) SC_STEP(3, a7) SC_STEP(2, a1)
  SC_STEP(5, a3) SC_STEP(4, a3) SC_STEP(2, a1) SC_STEP(8, a3) SC_STEP(3, a3) SC_STEP(3, a1)
  SC_STEP(6, a1) SC_STEP(5, a7) SC_STEP(3, a7)
#undef SC_STEP
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = t[i];
}
// a > (n-1)/2 ?
KGV_HD bool sc_is_high(const uint32_t* a) {
  const uint32_t hn[8] = {0x681B20A0u, 0xDFE92F46u, 0x57A4501Du, 0x5D576E73u, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0x7FFFFFFFu};
  return lt8(hn, a);
}

// r[0..4] = (a[0..4] * b[0..4]) mod 2^160   (15 partial products)
KGV_HD void mul_trunc5(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int i = 0; i < 5; i++) r[i] = 0;
#pragma unroll
  for (int i = 0; i < 5; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j + i < 5; j++) {
      uint64_t t = (uint64_t)a[i] * b[j] + r[i + j] + c;
      r[i + j] = (uint32_t)t;
      c = t >> 32;
    }
  }
}

// 160-bit two's complement helpers (5 limbs)
KGV_HD void sub5(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint64_t br = 0;
#pragma unroll
  for (int i = 0; i < 5; i++) {
    uint64_t t = (uint64_t)a[i] - b[i] - br;
    r[i] = (uint32_t)t;
    br = (t >> 32) & 1;
  }
}
KGV_HD void neg5(uint32_t* r) {
  uint64_t c = 1;
#pragma unroll
  for (int i = 0; i < 5; i++) {
    c += (uint32_t)~r[i];
    r[i] = (uint32_t)c;
    c >>= 32;
  }
}

// GLV split: k (mod n, 8 limbs) -> |k1|, |k2| (5 limbs each, < 2^128 in practice) and their signs,
// with k == s1*|k1| + s2*|k2|*lambda (mod n).  Pure integer arithmetic (no modular reduction):
//   c1 = round(k*g1 / 2^384), c2 = round(k*g2 / 2^384)
//   k1 = k - c1*a1 - c2*a2,  k2 = c1*|b1| - c2*b2      (both tiny, evaluated mod 2^160)
KGV_HD void glv_split(uint32_t* k1, bool& neg1, uint32_t* k2, bool& neg2, const uint32_t* k) {
  const uint32_t g1[8] = KGV_G1_LIMBS, g2[8] = KGV_G2_LIMBS;
  const uint32_t a1[5] = KGV_A1_LIMBS, mb1[5] = KGV_MB1_LIMBS, a2[5] = KGV_A2_LIMBS;
  uint32_t t[16], c1[5], c2[5];
  mul_wide(t, k, g1);
  {
    uint64_t c = (t[11] >> 31);
#pragma unroll
    for (int i = 0; i < 4; i++) { c += t[12 + i]; c1[i] = (uint32_t)c; c >>= 32; }
    c1[4] = (uint32_t)c;
  }
  mul_wide(t, k, g2);
  {
    uint64_t c = (t[11] >> 31);
#pragma unroll
    for (int i = 0; i < 4; i++) { c += t[12 + i]; c2[i] = (uint32_t)c; c >>= 32; }
    c2[4] = (uint32_t)c;
  }
  uint32_t p1[5], p2[5];
  // k1 = k - c1*a1 - c2*a2  (mod 2^160)
  mul_trunc5(p1, c1, a1);
  mul_trunc5(p2, c2, a2);
  sub5(k1, k, p1);
  sub5(k1, k1, p2);
  // k2 = c1*|b1| - c2*b2  (b2 == a1)
  mul_trunc5(p1, c1, mb1);
  mul_trunc5(p2, c2, a1);
  sub5(k2, p1, p2);
  neg1 = (k1[4] >> 31) != 0;
  if (neg1) neg5(k1);
  neg2 = (k2[4] >> 31) != 0;
  if (neg2) neg5(k2);
}

// Signed odd-digit recoding of a magnitude m < 2^131 (5 limbs).
// If m is even it is replaced by m+1 and `fix` is set (caller subtracts one table base point).
// Then m = sum_{i=0}^{32} d_i 16^i with every d_i odd in {+-1,..,+-15}:
//   h = (m >> 1) | 2^131 ; v_i = (h >> 4i) & 15 ; d_i = 2 v_i - 15.
KGV_HD void recode_signed_odd(uint32_t* h, bool& fix, const uint32_t* m) {
  uint32_t t[5];
  fix = (m[0] & 1u) == 0;
  uint64_t c = fix ? 1 : 0;
#pragma unroll
  for (int i = 0; i < 5; i++) { c += m[i]; t[i] = (uint32_t)c; c >>= 32; }
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = (t[i] >> 1) | (t[i + 1] << 31);
  h[4] = (t[4] >> 1) | (1u << 3);  // bit 131 = bit 3 of limb 4
}
// digit i (0..32) of a recoded scalar: table index 0..7 ((|d|-1)/2) and sign
KGV_HD void recoded_digit(const uint32_t* h, int i, uint32_t& idx, bool& neg) {
  uint32_t v = (h[i >> 3] >> ((i & 7) * 4)) & 15u;
  neg = (v & 8u) == 0;
  idx = neg ? (~v & 7u) : (v & 7u);
}

// ------------------------------------------------------------------------------------------
// group law, Jacobian coordinates on y^2 = x^3 + b (a = 0; b never appears in the formulas,
// so the same code runs on the isomorphic curves used for the per-thread tables)
// ------------------------------------------------------------------------------------------
// r = 2r for a finite r (callers test r.inf).  Each sum between the products is one wide accumulator (fex) with a
// single fold (fe_fold) at the end.
KGV_HD void gej_double_body(gej& r) {
  fe A, B, C, D, E, t;
  fex w, c8;
  fe_sqr(A, r.x);
  fe_sqr(B, r.y);
  fe_sqr(C, B);
  fe_add(t, r.x, B);
  fe_sqr(t, t);
  fex_set(w, t); fex_sub(w, A); fex_sub(w, C); fex_shl(w, 1);
  fe_fold(D, w);                        // D = 2((X+B)^2 - A - C) = 4 X Y^2
  fex_set(w, A); fex_shl(w, 1); fex_add(w, A);
  fe_fold(E, w);                        // E = 3 X^2
  fe_mul(t, r.y, r.z);
  fex_set(w, t); fex_shl(w, 1);
  fe_fold(r.z, w);                      // Z3 = 2 Y Z
  fe_sqr(t, E);
  fex_set(w, t); fex_sub(w, D); fex_sub(w, D);
  fe_fold(r.x, w);                      // X3 = E^2 - 2D
  fe_sub(t, D, r.x);
  fe_mul(t, E, t);
  fex_set(c8, C); fex_shl(c8, 3);
  fex_set(w, t); fex_sub_x(w, c8);
  fe_fold(r.y, w);                      // Y3 = E (D - X3) - 8 Y^4
}

// r += (bx,by) with the addend affine and never the point at infinity.  Handles r = inf and r == -addend (result
// infinity); for r == addend it leaves r as it is and returns true: the caller doubles r.  If hout != nullptr it
// receives the factor by which Z was multiplied (H), used by the table builder.
KGV_HD bool gej_add_ge_body(gej& r, const fe& bx, const fe& by, fe* hout) {
  if (r.inf) {
    r.x = bx;
    r.y = by;
    fe_set_u32(r.z, 1);
    r.inf = false;
    if (hout) fe_set_u32(*hout, 1);
    return false;
  }
  fe z1z1, u2, s2, h, rr, t;
  fe_sqr(z1z1, r.z);
  fe_mul(u2, bx, z1z1);
  fe_mul(t, r.z, z1z1);
  fe_mul(s2, by, t);
  fe_sub(h, u2, r.x);
  fe_sub(rr, s2, r.y);
  if (fe_is_zero(h)) {
    if (fe_is_zero(rr)) return true;
    if (hout) fe_set_u32(*hout, 1);
    r.inf = true;
    return false;
  }
  if (hout) *hout = h;
  fe hh, hhh, v;
  fex w;
  fe_sqr(hh, h);
  fe_mul(hhh, hh, h);
  fe_mul(v, r.x, hh);
  fe_mul(r.z, r.z, h);
  fe_sqr(t, rr);
  fex_set(w, t); fex_sub(w, hhh); fex_sub(w, v); fex_sub(w, v);
  fe_fold(r.x, w);        // X3 = R^2 - H^3 - 2V
  fe_sub(t, v, r.x);
  fe_mul(t, rr, t);
  fe_mul(hhh, r.y, hhh);
  fe_sub(r.y, t, hhh);    // Y3 = R (V - X3) - Y1 H^3
  return false;
}

// On the device the whole group law is ONE non-inlined function taking and returning the point by value:
//  * n > 0: r = 2^n r - the ladder's four doublings per window cross the call ABI once, with r in registers;
//  * n == 0: r += (bx,by), also returning H (the table builder needs it; it used to take it from an INLINED body:
//    seven unrolled copies, ~160 KB of straight-line code that evicted the ladder's hot code, DESIGN.md §4 K1).
//    The rare r == addend case falls through into the same doubling loop: no second copy of the doubling, no call.
// The point at infinity is tested by the caller of a doubling, once per call, not inside the doubling.  The host unit-test build inlines it.
#if defined(__CUDACC__)
struct gej_h { gej r; fe h; };
static __device__ __noinline__ gej_h gej_point_call(gej r, fe bx, fe by, int n) {
  gej_h o;
  if (n == 0 && gej_add_ge_body(r, bx, by, &o.h)) {
    fe_dbl(o.h, r.y);  // Z3 = 2 Y1 Z1 (cannot happen in the table builder)
    n = 1;
  }
#pragma unroll 1
  for (int i = 0; i < n; i++) gej_double_body(r);
  o.r = r;
  return o;
}
KGV_HD void gej_double_n(gej& r, int n) {
  if (!r.inf) r = gej_point_call(r, r.x, r.y, n).r;  // (bx, by unused)
}
KGV_HD void gej_add_ge(gej& r, const fe& bx, const fe& by, fe* hout = nullptr) {
  gej_h o = gej_point_call(r, bx, by, 0);
  r = o.r;
  if (hout) *hout = o.h;
}
#else
KGV_HD void gej_double_n(gej& r, int n) {
  if (r.inf) return;
  for (int i = 0; i < n; i++) gej_double_body(r);
}
KGV_HD void gej_add_ge(gej& r, const fe& bx, const fe& by, fe* hout = nullptr) {
  if (gej_add_ge_body(r, bx, by, hout)) {
    if (hout) fe_dbl(*hout, r.y);
    gej_double_n(r, 1);
  }
}
#endif
KGV_HD void gej_double(gej& r) { gej_double_n(r, 1); }

// y^2 = x^3 + 7: solve for y with the requested parity.  false if x is not on the curve.
// x must be canonical (< p).
KGV_HD bool ge_lift_x(fe& y, const fe& x, bool odd) {
  fe t, c;
  fe_sqr(t, x);
  fe_mul(t, t, x);
  fe_set_u32(c, 7);
  fe_add(c, t, c);
  if (!fe_sqrt(y, c)) return false;
  fe_normalize(y);
  if (((y.v[0] & 1u) != 0) != odd) {
    fe_neg(y, y);
    fe_normalize(y);
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// per-thread table of odd multiples {1,3,...,15} * P, "effective affine"
// ------------------------------------------------------------------------------------------
// Tab is an accessor with  void put(int entry, int word, uint32_t v)  and  uint32_t get(int entry, int word)
// (entry 0..NE-1, word 0..15: x limbs then y limbs).
//
// After the call, entry j holds the affine coordinates of (2j+1)*P on the isomorphic curve
// E' : y^2 = x^3 + 7*zs^6, where zs (returned) is such that a Jacobian point (X,Y,Z) on E'
// corresponds to (X, Y, Z*zs) on secp256k1.  lambda*(entry) = (beta*x, y) also holds on E'.
// NE: the number of entries, 8 for the verify ladders; the comb-form record builds {1,3,5,7} * T per tooth (NE = 4).
template <int NE = 8, class Tab>
KGV_HD void build_odd_table(Tab& tab, fe& zs, const fe& px, const fe& py) {
  static_assert(NE >= 2 && NE <= 8, "build_odd_table: 2 to 8 entries");
  // D = 2P (from affine input)
  gej d;
  d.x = px; d.y = py; fe_set_u32(d.z, 1); d.inf = false;
  gej_double(d);
  // map P onto the curve where D is affine: (x * Zd^2, y * Zd^3)
  fe zd2, zd3;
  fe_sqr(zd2, d.z);
  fe_mul(zd3, zd2, d.z);
  gej t;
  fe_mul(t.x, px, zd2);
  fe_mul(t.y, py, zd3);
  fe_set_u32(t.z, 1);
  t.inf = false;
  fe H[NE - 1];
#pragma unroll
  for (int w = 0; w < 8; w++) { tab.put(0, w, t.x.v[w]); tab.put(0, 8 + w, t.y.v[w]); }
#pragma unroll
  for (int j = 1; j < NE; j++) {
    gej_add_ge(t, d.x, d.y, &H[j - 1]);
#pragma unroll
    for (int w = 0; w < 8; w++) { tab.put(j, w, t.x.v[w]); tab.put(j, 8 + w, t.y.v[w]); }
  }
  // bring every entry to the Z of the last one: entry j *= (Z_last/Z_j)^{2,3}, Z_last/Z_j = H_{j+1}...H_last
  fe acc = H[NE - 2];
#pragma unroll
  for (int j = NE - 2; j >= 0; j--) {
    if (j < NE - 2) fe_mul(acc, acc, H[j]);
    fe a2, a3, ex, ey;
    fe_sqr(a2, acc);
    fe_mul(a3, a2, acc);
#pragma unroll
    for (int w = 0; w < 8; w++) { ex.v[w] = tab.get(j, w); ey.v[w] = tab.get(j, 8 + w); }
    fe_mul(ex, ex, a2);
    fe_mul(ey, ey, a3);
#pragma unroll
    for (int w = 0; w < 8; w++) { tab.put(j, w, ex.v[w]); tab.put(j, 8 + w, ey.v[w]); }
  }
  // total Z scale back to secp256k1: Z_7 (on D's curve) * Zd
  fe_mul(zs, t.z, d.z);
}

// ------------------------------------------------------------------------------------------
// R = kP * P + kG * G     (result on the isomorphic curve; true Z = R.z * zs)
// ------------------------------------------------------------------------------------------
// tab, zs: P's odd-multiples table and its Z scale, as build_odd_table leaves them (built by the caller, or copied from a key record).
// gtab: [8][65536][16] u32 — table j holds the affine (x limbs, y limbs) of v*2^(32j)*G; entry 0 unused.  This ladder reads j = 0 and 4.
// GLoad is a functor  void operator()(fe& x, fe& y, const uint32_t* entry)  (vectorised loads on device).
template <class Tab, class GLoad, class Trace = NoTrace>
KGV_HD void ecmult_double(gej& R, const fe& zs, const uint32_t* kP, const uint32_t* kG, Tab& tab, const uint32_t* gtab, GLoad gload,
                          Trace trace = Trace()) {
  const fe beta = {KGV_BETA_LIMBS};
  uint32_t m1[5], m2[5], h1[5], h2[5];
  bool neg1, neg2, fix1, fix2;
  glv_split(m1, neg1, m2, neg2, kP);
  recode_signed_odd(h1, fix1, m1);
  recode_signed_odd(h2, fix2, m2);
  trace(10, m1, 5); trace(11, m2, 5);
  { uint32_t f[4] = {neg1, neg2, fix1, fix2}; trace(12, f, 4); }
  trace(13, zs.v, 8);
  { uint32_t e0[16]; for (int w = 0; w < 16; w++) e0[w] = tab.get(7, w); trace(14, e0, 16); }
  fe zs2, zs3;
  fe_sqr(zs2, zs);
  fe_mul(zs3, zs2, zs);

  R.inf = true;
  fe_set_zero(R.x); fe_set_zero(R.y); fe_set_zero(R.z);
  for (int i = 32; i >= 0; i--) {
    if (i != 32) gej_double_n(R, 4);
    uint32_t idx; bool dn;
    fe ex, ey;
    // k1 digit on P
    recoded_digit(h1, i, idx, dn);
#pragma unroll
    for (int w = 0; w < 8; w++) { ex.v[w] = tab.get(idx, w); ey.v[w] = tab.get(idx, 8 + w); }
    if (dn != neg1) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
    // k2 digit on lambda*P = (beta*x, y)
    recoded_digit(h2, i, idx, dn);
#pragma unroll
    for (int w = 0; w < 8; w++) { ex.v[w] = tab.get(idx, w); ey.v[w] = tab.get(idx, 8 + w); }
    fe_mul(ex, ex, beta);
    if (dn != neg2) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
    // generator part: 16-bit windows every 4th step
    if ((i & 3) == 0 && i < 32) {
      int w16 = i >> 2;  // 0..7
      uint32_t dlo = (kG[w16 >> 1] >> ((w16 & 1) * 16)) & 0xFFFFu;
      uint32_t dhi = (kG[4 + (w16 >> 1)] >> ((w16 & 1) * 16)) & 0xFFFFu;
      if (dlo) {
        gload(ex, ey, gtab + (size_t)dlo * 16);
        fe_mul(ex, ex, zs2);
        fe_mul(ey, ey, zs3);
        gej_add_ge(R, ex, ey);
      }
      if (dhi) {
        gload(ex, ey, gtab + ((size_t)4 * 65536 + dhi) * 16);
        fe_mul(ex, ex, zs2);
        fe_mul(ey, ey, zs3);
        gej_add_ge(R, ex, ey);
      }
    }
  }
  trace(15, R.x.v, 8); trace(16, R.y.v, 8); trace(17, R.z.v, 8);
  // parity corrections: m was replaced by m+1 => subtract one base point
  if (fix1) {
    fe ex, ey;
#pragma unroll
    for (int w = 0; w < 8; w++) { ex.v[w] = tab.get(0, w); ey.v[w] = tab.get(0, 8 + w); }
    if (!neg1) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
  if (fix2) {
    fe ex, ey;
#pragma unroll
    for (int w = 0; w < 8; w++) { ex.v[w] = tab.get(0, w); ey.v[w] = tab.get(0, 8 + w); }
    fe_mul(ex, ex, beta);
    if (!neg2) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
}

// ------------------------------------------------------------------------------------------
// R = kP * P + kG * G from a four-tooth comb of P     (result with true Z)
// ------------------------------------------------------------------------------------------
// rec: entry 8t + e (16 words at word 16(8t + e)) is (2e+1) * 2^(32t) * P, true affine (key_comb_build, kgv_verify.cuh).
// gtab: as for ecmult_double, all eight tables.
// Digit i (0..32) of a recoded GLV half weighs 16^i = 2^(32t) * 16^w with t = i / 8, w = i % 8, except the top digit (i = 32:
// t = 3, w = 8).  So the ladder runs windows w = 8..0 with four doublings between them and adds, at window w, digit 8t + w of both halves
// from tooth t (33 additions per half, as ecmult_double); the generator adds bits 32j + 16..32j + 31 of kG from table j at window 4
// and bits 32j..32j + 15 at window 0 (16 additions).  32 doublings instead of 128.
// The key entries are staged through the thread's Tab slot: slot s = 2t + half holds one entry; after the addition that consumes
// slot s, the copy of its entry for the next window starts (one commit group per slot and window), so each copy has seven additions and
// the window's doublings to land.  stage_wait returns once all but the 7 most recent groups have landed.  The defaults below copy
// synchronously (host build); the device's shared-memory table overloads them with cp.async (SmemTab, kgv_lib.cu).
template <class Tab>
KGV_HD void stage_fetch(Tab& tab, int s, const uint32_t* entry) {
  for (int w = 0; w < 16; w++) tab.put(s, w, entry[w]);
}
template <class Tab>
KGV_HD void stage_commit(Tab&) {}
template <class Tab>
KGV_HD void stage_wait(Tab&) {}
template <class Tab>
KGV_HD void stage_get(Tab& tab, int s, fe& x, fe& y) {
  for (int w = 0; w < 8; w++) { x.v[w] = tab.get(s, w); y.v[w] = tab.get(s, 8 + w); }
}
KGV_HD const uint32_t* comb_entry(const uint32_t* rec, const uint32_t* h, int i, bool& neg) {
  uint32_t idx;
  recoded_digit(h, i, idx, neg);
  return rec + (8 * (i < 32 ? i >> 3 : 3) + idx) * 16;  // (the top digit: tooth 3)
}
template <class Tab, class GLoad>
KGV_HD void ecmult_comb(gej& R, const uint32_t* kP, const uint32_t* kG, const uint32_t* rec, Tab& tab, const uint32_t* gtab, GLoad gload) {
  const fe beta = {KGV_BETA_LIMBS};
  uint32_t m[2][5], h[2][5];
  bool ng[2], fix[2];
  glv_split(m[0], ng[0], m[1], ng[1], kP);
  recode_signed_odd(h[0], fix[0], m[0]);
  recode_signed_odd(h[1], fix[1], m[1]);
  bool dn;
#pragma unroll 1
  for (int s = 0; s < 8; s++) {
    stage_fetch(tab, s, comb_entry(rec, h[s & 1], 8 * (s >> 1) + 7, dn));
    stage_commit(tab);
  }
  R.inf = true;
  fe_set_zero(R.x); fe_set_zero(R.y); fe_set_zero(R.z);
  fe ex, ey;
  // window 8: the top digits, from tooth 3 (read directly while window 7's entries are on their way)
#pragma unroll 1
  for (int half = 0; half < 2; half++) {
    gload(ex, ey, comb_entry(rec, h[half], 32, dn));
    if (half) fe_mul(ex, ex, beta);
    if (dn != ng[half]) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
#pragma unroll 1
  for (int w = 7; w >= 0; w--) {
    gej_double_n(R, 4);
#pragma unroll 1
    for (int s = 0; s < 8; s++) {
      const int half = s & 1, i = 8 * (s >> 1) + w;
      uint32_t idx;
      recoded_digit(h[half], i, idx, dn);
      stage_wait(tab);
      stage_get(tab, s, ex, ey);
      if (half) fe_mul(ex, ex, beta);
      if (dn != ng[half]) fe_neg(ey, ey);
      gej_add_ge(R, ex, ey);
      bool dn1;
      if (w) stage_fetch(tab, s, comb_entry(rec, h[half], i - 1, dn1));
      stage_commit(tab);  // (empty in the last window: keeps stage_wait's count)
    }
    if ((w & 3) == 0) {
#pragma unroll 1
      for (int j = 0; j < 8; j++) {
        const uint32_t d = (kG[j] >> (w ? 16 : 0)) & 0xFFFFu;
        if (d) {
          gload(ex, ey, gtab + ((size_t)j * 65536 + d) * 16);
          gej_add_ge(R, ex, ey);
        }
      }
    }
  }
  // parity corrections as in ecmult_double: subtract P (entry 0 of tooth 0), resp. lambda*P
#pragma unroll 1
  for (int half = 0; half < 2; half++) {
    if (!fix[half]) continue;
    gload(ex, ey, rec);
    if (half) fe_mul(ex, ex, beta);
    if (!ng[half]) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
}

// ------------------------------------------------------------------------------------------
// R = kP * P + kG * G from the joint table of a comb record     (result with true Z)
// ------------------------------------------------------------------------------------------
// Joint recoding of one GLV half m (5 limbs), after the parity fix m -> m + 1 of an even m (`fix`, as recode_signed_odd):
//   m = sum_t c_t 2^(32t), t = 0..3, every c_t odd with |c_t| < 2^33: from the low tooth up, c_t = r mod 2^32, minus 2^32 (and one more
//   carry) when the quotient would be even, so every quotient stays odd; c_3 is the last quotient;
//   c_t = sum_w d_w 8^w, w = 0..10, d_w odd in {+-1, +-3, +-5, +-7}: v = (c_t + 2^33 - 1) / 2, d_w = 2 ((v >> 3w) & 7) - 7.
// glv_split's halves are below 2^128: |k1| <= (a1 + a2)/2 + 1 and |k2| <= (|b1| + b2)/2 + 1 (each rounding error of c1, c2 is at most
// 1/2 + 2^-128; a1 b2 - a2 b1 = n), and both bounds are below 2^128 (tests/test_hostsim_joint.py evaluates them).  So c_3 <= 2^32 + 1.
// Digit 11t + w is stored as the 3-bit v field in bits 3(i % 10) of word i / 10 (44 digits, 5 words).
KGV_HD void recode_joint(uint32_t* h, bool& fix, const uint32_t* m) {
  fix = (m[0] & 1u) == 0;
  uint64_t v[4], carry = fix ? 1 : 0;  // r_t = (m >> 32t) + carry, odd
#pragma unroll
  for (int t = 0; t < 3; t++) {
    const uint64_t x = (uint64_t)m[t] + carry;
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);  // lo: the low word of r_t, odd
    const uint32_t borrow = ((m[t + 1] + hi) & 1u) ^ 1u;         // the quotient would be even: c_t = lo - 2^32
    v[t] = (uint64_t)(lo >> 1) + (borrow ? (1ull << 31) : (1ull << 32));
    carry = hi + borrow;
  }
  const uint64_t c3 = (uint64_t)m[3] + ((uint64_t)m[4] << 32) + carry;  // odd, positive
  v[3] = (c3 >> 1) + (1ull << 32);
#pragma unroll
  for (int q = 0; q < 5; q++) h[q] = 0;
#pragma unroll
  for (int i = 0; i < 44; i++) h[i / 10] |= (uint32_t)((v[i / 11] >> (3 * (i % 11))) & 7u) << (3 * (i % 10));
}
// the v field (0..7, d = 2v - 7) of digit i = 11t + w
KGV_HD uint32_t joint_digit(const uint32_t* h, int i) { return (h[i / 10] >> (3 * (i % 10))) & 7u; }
// jt: the joint table, entry 32t + 8a + k (16 words at word 16(32t + 8a + k)) = (2a+1) T + (2k-7) lambda T, T = 2^(32t) P, true affine
// (joint_table_build, kgv_verify.cuh).  The entry for digit i of both halves, with the GLV signs ng folded in: e0 T + e1 lambda T =
// sign(e0) (|e0| T + sign(e0) e1 lambda T); neg: negate its y.
KGV_HD const uint32_t* joint_entry(const uint32_t* jt, const uint32_t (*h)[5], const bool* ng, int i, bool& neg) {
  const uint32_t u0 = joint_digit(h[0], i), u1 = joint_digit(h[1], i);
  neg = (u0 < 4u) != ng[0];
  const uint32_t a = u0 < 4u ? 3u - u0 : u0 - 4u;   // (|d0| - 1) / 2
  const uint32_t k = neg != ng[1] ? 7u - u1 : u1;   // b = sign(e0) e1 = 2k - 7
  return jt + 16 * (32 * (i / 11) + 8 * a + k);
}
// the eight generator additions of 16-bit fields at bits 32j + sh of kG, from table j (zero fields skipped)
template <class GLoad>
KGV_HD void gen_fields(gej& R, const uint32_t* kG, int sh, const uint32_t* gtab, GLoad gload) {
  fe ex, ey;
#pragma unroll 1
  for (int j = 0; j < 8; j++) {
    const uint32_t d = (kG[j] >> sh) & 0xFFFFu;
    if (d) {
      gload(ex, ey, gtab + ((size_t)j * 65536 + d) * 16);
      gej_add_ge(R, ex, ey);
    }
  }
}
// rec: a record whose first 16 words are P, true affine (the comb-form record, KGV_JR_*, or the reference comb record, KGV_KC_*: entry 0);
// jt: its joint table.  gtab: as for ecmult_comb.
// Windows w = 10..0 with three doublings between them (30 in all); window w adds, per tooth t, ONE joint entry for digit 11t + w of both
// halves (44 key additions, no beta products).  The generator's fields at bits 32j..32j+15 weigh 1 (after window 0); those at bits
// 32j+16..32j+31 weigh 2^16 = 2 * 2^(3*5): window 5's three doublings are split 2 + 1 around them.  Both use the eight tables of ecmult_comb
// (32 MiB, L2 resident), none more.
// Staging as in ecmult_comb: window 10 is read directly; window w's entry of tooth t sits in slot 4(w & 1) + t; after the addition that
// consumes it, the copy of the entry of window w - 2 starts into the same slot (one commit group per addition, empty ones in windows 1, 0).
// Between a copy's commit and its read lie 3 - t + 4 + t = 7 newer groups: stage_wait's count.
template <class Tab, class GLoad>
KGV_HD void ecmult_joint(gej& R, const uint32_t* kP, const uint32_t* kG, const uint32_t* rec, const uint32_t* jt, Tab& tab, const uint32_t* gtab,
                         GLoad gload) {
  const fe beta = {KGV_BETA_LIMBS};
  uint32_t m[2][5], h[2][5];
  bool ng[2], fix[2], neg;
  glv_split(m[0], ng[0], m[1], ng[1], kP);
  recode_joint(h[0], fix[0], m[0]);
  recode_joint(h[1], fix[1], m[1]);
#pragma unroll 1
  for (int s = 0; s < 8; s++) {  // window 9 into slots 4..7, then window 8 into slots 0..3
    const int w = 9 - (s >> 2), t = s & 3;
    stage_fetch(tab, 4 * (w & 1) + t, joint_entry(jt, h, ng, 11 * t + w, neg));
    stage_commit(tab);
  }
  R.inf = true;
  fe_set_zero(R.x); fe_set_zero(R.y); fe_set_zero(R.z);
  fe ex, ey;
#pragma unroll 1
  for (int t = 0; t < 4; t++) {
    gload(ex, ey, joint_entry(jt, h, ng, 11 * t + 10, neg));
    if (neg) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
#pragma unroll 1
  for (int w = 9; w >= 0; w--) {
    if (w == 5) {
      gej_double_n(R, 2);
      gen_fields(R, kG, 16, gtab, gload);
      gej_double_n(R, 1);
    } else {
      gej_double_n(R, 3);
    }
#pragma unroll 1
    for (int t = 0; t < 4; t++) {
      const int s = 4 * (w & 1) + t;
      (void)joint_entry(jt, h, ng, 11 * t + w, neg);
      stage_wait(tab);
      stage_get(tab, s, ex, ey);
      if (neg) fe_neg(ey, ey);
      gej_add_ge(R, ex, ey);
      bool neg2;
      if (w >= 2) stage_fetch(tab, s, joint_entry(jt, h, ng, 11 * t + w - 2, neg2));
      stage_commit(tab);  // (empty in windows 1 and 0: keeps stage_wait's count)
    }
  }
  gen_fields(R, kG, 0, gtab, gload);
  // parity corrections, at most one addition: -(s0 P + s1 lambda P) = -s0 (P + s0 s1 lambda P) is joint entry (a = 1, b = s0 s1) of
  // tooth 0; one of them alone is P (rec's first 16 words), times beta for the lambda half
  if (fix[0] && fix[1]) {
    gload(ex, ey, jt + 16 * (ng[0] == ng[1] ? 4 : 3));
    if (!ng[0]) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  } else if (fix[0] || fix[1]) {
    const int half = fix[1] ? 1 : 0;
    gload(ex, ey, rec);
    if (half) fe_mul(ex, ex, beta);
    if (!ng[half]) fe_neg(ey, ey);
    gej_add_ge(R, ex, ey);
  }
}

}  // namespace kgv
