// kgv_arith.cuh — 256-bit limb primitives and secp256k1 field arithmetic for sm_90a.
//
// One number per thread, 8 x 32-bit little-endian limbs held in registers.  Products are
// built from IMAD.WIDE.U32(.X) carry chains (mad.lo.cc / madc.hi.cc pairs, which ptxas fuses
// into one IMAD.WIDE.U32.X each); tools/microbench/pipes.cu and femul.cu measure what an IMAD.WIDE
// and an IADD3 cost per warp instruction per SM sub-partition.
//
// Replaces, for the GPU path, the field arithmetic of the C libsecp256k1 that the reference
// reaches through crypto/txscript/src/lib.rs:593 / :628 (`sig.verify`).
//
// Every function is KGV_HD so that tests/hostsim can compile the same logic for the host with
// the portable (non-PTX) primitive bodies and unit-test it on a GPU-less machine.  The host
// bodies exist only for that test build: the shipped library has no CPU execution path.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
// Under nvcc everything here is device-only code; the plain-C++ bodies below exist only for the
// host unit-test build in tests/hostsim (compiled by g++, never linked into the product).
#define KGV_HD __device__ __forceinline__
#define KGV_D __device__ __forceinline__
#else
#define KGV_HD inline
#define KGV_D inline
#endif

namespace kgv {

// ---------------------------------------------------------------------------------------------
// carry-chain primitives
// ---------------------------------------------------------------------------------------------

// r = a + b (8 limbs); returns the carry out (0/1)
KGV_HD uint32_t add8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %9, %17;\n\t"
      "addc.cc.u32 %1, %10, %18;\n\t"
      "addc.cc.u32 %2, %11, %19;\n\t"
      "addc.cc.u32 %3, %12, %20;\n\t"
      "addc.cc.u32 %4, %13, %21;\n\t"
      "addc.cc.u32 %5, %14, %22;\n\t"
      "addc.cc.u32 %6, %15, %23;\n\t"
      "addc.cc.u32 %7, %16, %24;\n\t"
      "addc.u32 %8, 0, 0;"
      : "=&r"(r[0]), "=&r"(r[1]), "=&r"(r[2]), "=&r"(r[3]), "=&r"(r[4]), "=&r"(r[5]), "=&r"(r[6]), "=&r"(r[7]), "=&r"(c)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]), "r"(b[0]), "r"(b[1]), "r"(b[2]),
        "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
#else
  uint64_t t = 0;
  for (int i = 0; i < 8; i++) { t += (uint64_t)a[i] + b[i]; r[i] = (uint32_t)t; t >>= 32; }
  c = (uint32_t)t;
#endif
  return c;
}

// r = a - b (8 limbs); returns the borrow out (0/1)
KGV_HD uint32_t sub8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t bo;
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %9, %17;\n\t"
      "subc.cc.u32 %1, %10, %18;\n\t"
      "subc.cc.u32 %2, %11, %19;\n\t"
      "subc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\t"
      "subc.cc.u32 %5, %14, %22;\n\t"
      "subc.cc.u32 %6, %15, %23;\n\t"
      "subc.cc.u32 %7, %16, %24;\n\t"
      "subc.u32 %8, 0, 0;"
      : "=&r"(r[0]), "=&r"(r[1]), "=&r"(r[2]), "=&r"(r[3]), "=&r"(r[4]), "=&r"(r[5]), "=&r"(r[6]), "=&r"(r[7]), "=&r"(bo)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]), "r"(b[0]), "r"(b[1]), "r"(b[2]),
        "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
  bo &= 1u;  // subc of 0-0-borrow yields 0 or 0xFFFFFFFF
#else
  uint64_t br = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t t = (uint64_t)a[i] - b[i] - br;
    r[i] = (uint32_t)t;
    br = (t >> 32) & 1;
  }
  bo = (uint32_t)br;
#endif
  return bo;
}

// r += (a2:a1:a0) at limb 0, propagating through all 8 limbs; returns carry out
KGV_HD uint32_t add8_small3(uint32_t* r, uint32_t a0, uint32_t a1, uint32_t a2) {
  uint32_t c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %9;\n\t"
      "addc.cc.u32 %1, %1, %10;\n\t"
      "addc.cc.u32 %2, %2, %11;\n\t"
      "addc.cc.u32 %3, %3, 0;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "addc.cc.u32 %6, %6, 0;\n\t"
      "addc.cc.u32 %7, %7, 0;\n\t"
      "addc.u32 %8, 0, 0;"
      : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]), "=r"(c)
      : "r"(a0), "r"(a1), "r"(a2));
#else
  uint64_t t = (uint64_t)r[0] + a0; r[0] = (uint32_t)t; t >>= 32;
  t += (uint64_t)r[1] + a1; r[1] = (uint32_t)t; t >>= 32;
  t += (uint64_t)r[2] + a2; r[2] = (uint32_t)t; t >>= 32;
  for (int i = 3; i < 8; i++) { t += r[i]; r[i] = (uint32_t)t; t >>= 32; }
  c = (uint32_t)t;
#endif
  return c;
}

// r -= (a1:a0) at limb 0, propagating through all 8 limbs; returns borrow out
KGV_HD uint32_t sub8_small2(uint32_t* r, uint32_t a0, uint32_t a1) {
  uint32_t bo;
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %0, %9;\n\t"
      "subc.cc.u32 %1, %1, %10;\n\t"
      "subc.cc.u32 %2, %2, 0;\n\t"
      "subc.cc.u32 %3, %3, 0;\n\t"
      "subc.cc.u32 %4, %4, 0;\n\t"
      "subc.cc.u32 %5, %5, 0;\n\t"
      "subc.cc.u32 %6, %6, 0;\n\t"
      "subc.cc.u32 %7, %7, 0;\n\t"
      "subc.u32 %8, 0, 0;"
      : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]), "=r"(bo)
      : "r"(a0), "r"(a1));
  bo &= 1u;
#else
  uint64_t br = 0, t;
  t = (uint64_t)r[0] - a0; r[0] = (uint32_t)t; br = (t >> 32) & 1;
  t = (uint64_t)r[1] - a1 - br; r[1] = (uint32_t)t; br = (t >> 32) & 1;
  for (int i = 2; i < 8; i++) { t = (uint64_t)r[i] - br; r[i] = (uint32_t)t; br = (t >> 32) & 1; }
  bo = (uint32_t)br;
#endif
  return bo;
}

// x[0..7] += a0*b + (a1*b << 64) + (a2*b << 128) + (a3*b << 192); carry out is added into x[8].
// One carry chain of four IMAD.WIDE.U32.X plus one IADD3.X.
KGV_HD void mad_row4(uint32_t* x, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b) {
#if defined(__CUDACC__)
  asm("mad.lo.cc.u32  %0, %9, %13, %0;\n\t"
      "madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
      "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
      "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
      "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
      "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
      "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
      "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(x[8])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b));
#else
  const uint32_t a[4] = {a0, a1, a2, a3};
  uint64_t c = 0;
  for (int j = 0; j < 4; j++) {
    uint64_t p = (uint64_t)a[j] * b;
    uint64_t lo = (uint64_t)x[2 * j] + (uint32_t)p + c;
    x[2 * j] = (uint32_t)lo;
    uint64_t hi = (uint64_t)x[2 * j + 1] + (uint32_t)(p >> 32) + (lo >> 32);
    x[2 * j + 1] = (uint32_t)hi;
    c = hi >> 32;
  }
  x[8] += (uint32_t)c;
#endif
}

// 3-product variant of mad_row4: x[0..5] += sum a_j*b << 64j ; carry out added into x[6]
KGV_HD void mad_row3(uint32_t* x, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t b) {
#if defined(__CUDACC__)
  asm(
      "mad.lo.cc.u32  %0, %7, %10, %0;\n\t"
      "madc.hi.cc.u32 %1, %7, %10, %1;\n\t"
      "madc.lo.cc.u32 %2, %8, %10, %2;\n\t"
      "madc.hi.cc.u32 %3, %8, %10, %3;\n\t"
      "madc.lo.cc.u32 %4, %9, %10, %4;\n\t"
      "madc.hi.cc.u32 %5, %9, %10, %5;\n\t"
      "addc.u32 %6, %6, 0;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6])
      : "r"(a0), "r"(a1), "r"(a2), "r"(b));
#else
  const uint32_t a[3] = {a0, a1, a2};
  uint64_t c = 0;
  for (int j = 0; j < 3; j++) {
    uint64_t p = (uint64_t)a[j] * b;
    uint64_t lo = (uint64_t)x[2 * j] + (uint32_t)p + c;
    x[2 * j] = (uint32_t)lo;
    uint64_t hi = (uint64_t)x[2 * j + 1] + (uint32_t)(p >> 32) + (lo >> 32);
    x[2 * j + 1] = (uint32_t)hi;
    c = hi >> 32;
  }
  x[6] += (uint32_t)c;
#endif
}

// 2-product variant of mad_row4: x[0..3] += sum a_j*b << 64j ; carry out added into x[4]
KGV_HD void mad_row2(uint32_t* x, uint32_t a0, uint32_t a1, uint32_t b) {
#if defined(__CUDACC__)
  asm(
      "mad.lo.cc.u32  %0, %5, %7, %0;\n\t"
      "madc.hi.cc.u32 %1, %5, %7, %1;\n\t"
      "madc.lo.cc.u32 %2, %6, %7, %2;\n\t"
      "madc.hi.cc.u32 %3, %6, %7, %3;\n\t"
      "addc.u32 %4, %4, 0;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4])
      : "r"(a0), "r"(a1), "r"(b));
#else
  const uint32_t a[2] = {a0, a1};
  uint64_t c = 0;
  for (int j = 0; j < 2; j++) {
    uint64_t p = (uint64_t)a[j] * b;
    uint64_t lo = (uint64_t)x[2 * j] + (uint32_t)p + c;
    x[2 * j] = (uint32_t)lo;
    uint64_t hi = (uint64_t)x[2 * j + 1] + (uint32_t)(p >> 32) + (lo >> 32);
    x[2 * j + 1] = (uint32_t)hi;
    c = hi >> 32;
  }
  x[4] += (uint32_t)c;
#endif
}

// 1-product variant of mad_row4: x[0..1] += sum a_j*b << 64j ; carry out added into x[2]
KGV_HD void mad_row1(uint32_t* x, uint32_t a0, uint32_t b) {
#if defined(__CUDACC__)
  asm(
      "mad.lo.cc.u32  %0, %3, %4, %0;\n\t"
      "madc.hi.cc.u32 %1, %3, %4, %1;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2])
      : "r"(a0), "r"(b));
#else
  const uint32_t a[1] = {a0};
  uint64_t c = 0;
  for (int j = 0; j < 1; j++) {
    uint64_t p = (uint64_t)a[j] * b;
    uint64_t lo = (uint64_t)x[2 * j] + (uint32_t)p + c;
    x[2 * j] = (uint32_t)lo;
    uint64_t hi = (uint64_t)x[2 * j + 1] + (uint32_t)(p >> 32) + (lo >> 32);
    x[2 * j + 1] = (uint32_t)hi;
    c = hi >> 32;
  }
  x[2] += (uint32_t)c;
#endif
}

// t[0..15] = e[0..15] + (o[0..14] << 32): recombine the even/odd column accumulators
KGV_HD void merge_eo(uint32_t* t, const uint32_t* e, const uint32_t* o) {
  t[0] = e[0];
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %15, %30;\n\t"
      "addc.cc.u32 %1, %16, %31;\n\t"
      "addc.cc.u32 %2, %17, %32;\n\t"
      "addc.cc.u32 %3, %18, %33;\n\t"
      "addc.cc.u32 %4, %19, %34;\n\t"
      "addc.cc.u32 %5, %20, %35;\n\t"
      "addc.cc.u32 %6, %21, %36;\n\t"
      "addc.cc.u32 %7, %22, %37;\n\t"
      "addc.cc.u32 %8, %23, %38;\n\t"
      "addc.cc.u32 %9, %24, %39;\n\t"
      "addc.cc.u32 %10, %25, %40;\n\t"
      "addc.cc.u32 %11, %26, %41;\n\t"
      "addc.cc.u32 %12, %27, %42;\n\t"
      "addc.cc.u32 %13, %28, %43;\n\t"
      "addc.u32 %14, %29, %44;"
      : "=&r"(t[1]), "=&r"(t[2]), "=&r"(t[3]), "=&r"(t[4]), "=&r"(t[5]), "=&r"(t[6]), "=&r"(t[7]), "=&r"(t[8]), "=&r"(t[9]), "=&r"(t[10]),
        "=&r"(t[11]), "=&r"(t[12]), "=&r"(t[13]), "=&r"(t[14]), "=&r"(t[15])
      : "r"(e[1]), "r"(e[2]), "r"(e[3]), "r"(e[4]), "r"(e[5]), "r"(e[6]), "r"(e[7]), "r"(e[8]), "r"(e[9]), "r"(e[10]), "r"(e[11]),
        "r"(e[12]), "r"(e[13]), "r"(e[14]), "r"(e[15]), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]), "r"(o[4]), "r"(o[5]), "r"(o[6]),
        "r"(o[7]), "r"(o[8]), "r"(o[9]), "r"(o[10]), "r"(o[11]), "r"(o[12]), "r"(o[13]), "r"(o[14]));
#else
  uint64_t c = 0;
  for (int i = 1; i < 16; i++) { c += (uint64_t)e[i] + o[i - 1]; t[i] = (uint32_t)c; c >>= 32; }
#endif
}

// t[0..15] = a * b  (full 512-bit product).
// Even/odd column split: products whose limb position i+j is even accumulate in `e`, the others in
// `o` (which is the value shifted left by 32 bits), so every IMAD.WIDE lands on an aligned 64-bit
// register pair and each row is a single carry chain.  64 IMAD.WIDE + 16 IADD3.X + 15-limb merge.
KGV_HD void mul_wide(uint32_t* t, const uint32_t* a, const uint32_t* b) {
  uint32_t e[18], o[18];
#pragma unroll
  for (int i = 0; i < 18; i++) { e[i] = 0; o[i] = 0; }
#pragma unroll
  for (int i = 0; i < 8; i += 2) {
    // row i (even): a_even*b_i at even limbs i+j -> e ; a_odd*b_i at odd limbs i+j -> o[i+j-1]
    mad_row4(e + i, a[0], a[2], a[4], a[6], b[i]);
    mad_row4(o + i, a[1], a[3], a[5], a[7], b[i]);
    // row i+1 (odd): a_even*b at odd limbs -> o[i+1+j-1] ; a_odd*b at even limbs i+1+j -> e
    mad_row4(o + i, a[0], a[2], a[4], a[6], b[i + 1]);
    mad_row4(e + i + 2, a[1], a[3], a[5], a[7], b[i + 1]);
  }
  merge_eo(t, e, o);
}

// ---------------------------------------------------------------------------------------------
// field arithmetic modulo p = 2^256 - 2^32 - 977
// Elements are "weakly reduced": any representative in [0, 2^256).  fe_normalize gives the
// canonical one; comparisons and parity must normalize first.
// ---------------------------------------------------------------------------------------------
struct fe { uint32_t v[8]; };

#define KGV_P0 0xFFFFFC2Fu
#define KGV_P1 0xFFFFFFFEu

KGV_HD void fe_set_zero(fe& r) {
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = 0;
}
KGV_HD void fe_set_u32(fe& r, uint32_t x) { fe_set_zero(r); r.v[0] = x; }

// r += k * (2^32 + 977) for k in {0,1}; returns carry out
KGV_HD uint32_t fe_add_kC(fe& r, uint32_t k) { return add8_small3(r.v, 977u * k, k, 0u); }

// r[3..7] += 1 / r[3..7] -= 1; returns the carry / borrow out.  The rare tails of add_low2_rare, sub_low2_rare and
// fe_fold: one straight carry chain, so the untaken path stays short in the hot code.
KGV_HD uint32_t inc_hi5(uint32_t* r) {
  uint32_t c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, 1;\n\t"
      "addc.cc.u32 %1, %1, 0;\n\t"
      "addc.cc.u32 %2, %2, 0;\n\t"
      "addc.cc.u32 %3, %3, 0;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.u32 %5, 0, 0;"
      : "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]), "=r"(c));
#else
  uint64_t t = 1;
  for (int i = 3; i < 8; i++) { t += r[i]; r[i] = (uint32_t)t; t >>= 32; }
  c = (uint32_t)t;
#endif
  return c;
}
KGV_HD uint32_t dec_hi5(uint32_t* r) {
  uint32_t bo;
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %0, 1;\n\t"
      "subc.cc.u32 %1, %1, 0;\n\t"
      "subc.cc.u32 %2, %2, 0;\n\t"
      "subc.cc.u32 %3, %3, 0;\n\t"
      "subc.cc.u32 %4, %4, 0;\n\t"
      "subc.u32 %5, 0, 0;"
      : "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]), "=r"(bo));
  bo &= 1u;
#else
  uint64_t br = 1;
  for (int i = 3; i < 8; i++) {
    uint64_t t = (uint64_t)r[i] - br;
    r[i] = (uint32_t)t;
    br = (t >> 32) & 1;
  }
  bo = (uint32_t)br;
#endif
  return bo;
}

// r += (a1:a0) where the carry almost never leaves limb 2: three-limb chain, the (probability 2^-32)
// propagation through the upper limbs sits on a separate, normally untaken path.  Returns the carry out.
KGV_HD uint32_t add_low2_rare(uint32_t* r, uint32_t a0, uint32_t a1) {
  uint32_t c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %4;\n\t"
      "addc.cc.u32 %1, %1, %5;\n\t"
      "addc.cc.u32 %2, %2, 0;\n\t"
      "addc.u32 %3, 0, 0;"
      : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "=r"(c)
      : "r"(a0), "r"(a1));
#else
  uint64_t t = (uint64_t)r[0] + a0; r[0] = (uint32_t)t; t >>= 32;
  t += (uint64_t)r[1] + a1; r[1] = (uint32_t)t; t >>= 32;
  t += (uint64_t)r[2]; r[2] = (uint32_t)t; t >>= 32;
  c = (uint32_t)t;
#endif
  if (c) c = inc_hi5(r);
  return c;
}
// r -= (a1:a0), same structure; returns the borrow out
KGV_HD uint32_t sub_low2_rare(uint32_t* r, uint32_t a0, uint32_t a1) {
  uint32_t bo;
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %0, %4;\n\t"
      "subc.cc.u32 %1, %1, %5;\n\t"
      "subc.cc.u32 %2, %2, 0;\n\t"
      "subc.u32 %3, 0, 0;"
      : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "=r"(bo)
      : "r"(a0), "r"(a1));
  bo &= 1u;
#else
  uint64_t t = (uint64_t)r[0] - a0; r[0] = (uint32_t)t; uint64_t br = (t >> 32) & 1;
  t = (uint64_t)r[1] - a1 - br; r[1] = (uint32_t)t; br = (t >> 32) & 1;
  t = (uint64_t)r[2] - br; r[2] = (uint32_t)t; br = (t >> 32) & 1;
  bo = (uint32_t)br;
#endif
  if (bo) bo = dec_hi5(r);
  return bo;
}

KGV_HD void fe_add(fe& r, const fe& a, const fe& b) {
  uint32_t c = add8(r.v, a.v, b.v);
  c = add_low2_rare(r.v, 977u * c, c);   // 2^256 == C (mod p)
  if (c) (void)fe_add_kC(r, 1);          // only when the folded sum wrapped again (cannot wrap twice)
}

KGV_HD void fe_sub(fe& r, const fe& a, const fe& b) {
  uint32_t bo = sub8(r.v, a.v, b.v);
  bo = sub_low2_rare(r.v, 977u * bo, bo);  // -2^256 == -C (mod p)
  if (bo) (void)sub8_small2(r.v, 977u, 1u);
}

KGV_HD void fe_neg(fe& r, const fe& a) {
  fe z;
  fe_set_zero(z);
  fe_sub(r, z, a);
}

KGV_HD void fe_dbl(fe& r, const fe& a) { fe_add(r, a, a); }

// Wide accumulator for the additions around the group-law products: a 256-bit value plus a small signed multiple
// of 2^256 (|top| < 2^20, two's complement).  A whole sum such as 2((X+B)^2 - A - C) is one carry chain per operand
// into `top` and ONE fold (fe_fold) at the end, instead of a fold after every fe_add / fe_sub.
struct fex {
  uint32_t v[8];
  uint32_t top;
};
KGV_HD void fex_set(fex& r, const fe& a) {
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = a.v[i];
  r.top = 0;
}
// r += b
KGV_HD void fex_add(fex& r, const fe& b) {
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %9;\n\t"
      "addc.cc.u32 %1, %1, %10;\n\t"
      "addc.cc.u32 %2, %2, %11;\n\t"
      "addc.cc.u32 %3, %3, %12;\n\t"
      "addc.cc.u32 %4, %4, %13;\n\t"
      "addc.cc.u32 %5, %5, %14;\n\t"
      "addc.cc.u32 %6, %6, %15;\n\t"
      "addc.cc.u32 %7, %7, %16;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]), "+r"(r.top)
      : "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
#else
  uint64_t c = 0;
  for (int i = 0; i < 8; i++) { c += (uint64_t)r.v[i] + b.v[i]; r.v[i] = (uint32_t)c; c >>= 32; }
  r.top += (uint32_t)c;
#endif
}
// r -= b
KGV_HD void fex_sub(fex& r, const fe& b) {
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %0, %9;\n\t"
      "subc.cc.u32 %1, %1, %10;\n\t"
      "subc.cc.u32 %2, %2, %11;\n\t"
      "subc.cc.u32 %3, %3, %12;\n\t"
      "subc.cc.u32 %4, %4, %13;\n\t"
      "subc.cc.u32 %5, %5, %14;\n\t"
      "subc.cc.u32 %6, %6, %15;\n\t"
      "subc.cc.u32 %7, %7, %16;\n\t"
      "subc.u32 %8, %8, 0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]), "+r"(r.top)
      : "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
#else
  uint64_t br = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t t = (uint64_t)r.v[i] - b.v[i] - br;
    r.v[i] = (uint32_t)t;
    br = (t >> 32) & 1;
  }
  r.top -= (uint32_t)br;
#endif
}
// r -= b, both wide
KGV_HD void fex_sub_x(fex& r, const fex& b) {
#if defined(__CUDACC__)
  asm("sub.cc.u32 %0, %0, %9;\n\t"
      "subc.cc.u32 %1, %1, %10;\n\t"
      "subc.cc.u32 %2, %2, %11;\n\t"
      "subc.cc.u32 %3, %3, %12;\n\t"
      "subc.cc.u32 %4, %4, %13;\n\t"
      "subc.cc.u32 %5, %5, %14;\n\t"
      "subc.cc.u32 %6, %6, %15;\n\t"
      "subc.cc.u32 %7, %7, %16;\n\t"
      "subc.u32 %8, %8, %17;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]), "+r"(r.top)
      : "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]), "r"(b.top));
#else
  uint64_t br = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t t = (uint64_t)r.v[i] - b.v[i] - br;
    r.v[i] = (uint32_t)t;
    br = (t >> 32) & 1;
  }
  r.top = r.top - b.top - (uint32_t)br;
#endif
}
// r <<= k, 1 <= k <= 3
KGV_HD void fex_shl(fex& r, int k) {
#if defined(__CUDACC__)
  r.top = __funnelshift_l(r.v[7], r.top, k);
#pragma unroll
  for (int i = 7; i > 0; i--) r.v[i] = __funnelshift_l(r.v[i - 1], r.v[i], k);
#else
  r.top = (r.top << k) | (r.v[7] >> (32 - k));
  for (int i = 7; i > 0; i--) r.v[i] = (r.v[i] << k) | (r.v[i - 1] >> (32 - k));
#endif
  r.v[0] <<= k;
}
// r = a mod p, weakly reduced: a.v + top * 2^256 == a.v + top * (2^32 + 977).  top * (2^32 + 977) is a signed 96-bit
// addend (a0, a1, a2 sign-extended); after a three-limb chain the carry into limb 3 is -1, 0 or +1, and it is nonzero
// with probability ~2^-32 per unit of |top|: that propagation (and the wrap past 2^256 it may cause) sits on an
// untaken branch, like add_low2_rare.
KGV_HD void fe_fold(fe& r, const fex& a) {
  const int32_t top = (int32_t)a.top;
  const int32_t s = top * 977;
  const int32_t h = top + (s >> 31);  // top*C = (uint32)s + h * 2^32
  const uint32_t a0 = (uint32_t)s, a1 = (uint32_t)h, a2 = (uint32_t)(h >> 31);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = a.v[i];
  uint32_t c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %4;\n\t"
      "addc.cc.u32 %1, %1, %5;\n\t"
      "addc.cc.u32 %2, %2, %6;\n\t"
      "addc.u32 %3, 0, 0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "=r"(c)
      : "r"(a0), "r"(a1), "r"(a2));
#else
  {
    uint64_t t = (uint64_t)r.v[0] + a0; r.v[0] = (uint32_t)t; t >>= 32;
    t += (uint64_t)r.v[1] + a1; r.v[1] = (uint32_t)t; t >>= 32;
    t += (uint64_t)r.v[2] + a2; r.v[2] = (uint32_t)t; t >>= 32;
    c = (uint32_t)t;
  }
#endif
  const uint32_t net = c + a2;  // carry into limb 3 (a2 = 0xFFFFFFFF stands for -1): 0, 1 or 0xFFFFFFFF
  if (net != 0) {  // past 2^256 the rest is tiny (+1) or within 2^40 of 2^256 (-1): +-C cannot wrap again
    if (net == 1u) {
      if (inc_hi5(r.v)) (void)add8_small3(r.v, 977u, 1u, 0u);
    } else if (dec_hi5(r.v)) {
      (void)sub8_small2(r.v, 977u, 1u);
    }
  }
}

// canonical representative in [0, p)
KGV_HD void fe_normalize(fe& r) {
  // r >= p  <=>  r[2..7] all ones and (r[1]:r[0]) >= 0xFFFFFFFE_FFFFFC2F
  uint32_t hi = r.v[2] & r.v[3] & r.v[4] & r.v[5] & r.v[6] & r.v[7];
  bool ge = (hi == 0xFFFFFFFFu) && (r.v[1] == 0xFFFFFFFFu || (r.v[1] == KGV_P1 && r.v[0] >= KGV_P0));
  if (ge) {
    // r - p = r + C - 2^256 : only the low limbs survive
    (void)add8_small3(r.v, 977u, 1u, 0u);
  }
}
KGV_HD bool fe_is_zero_normalized(const fe& a) { return (a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7]) == 0; }
// is the (weakly reduced) element congruent to 0 ?  i.e. equal to 0 or to p
KGV_HD bool fe_is_zero(const fe& a) {
  uint32_t orv = a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7];
  uint32_t andv = a.v[2] & a.v[3] & a.v[4] & a.v[5] & a.v[6] & a.v[7];
  return orv == 0 || (andv == 0xFFFFFFFFu && a.v[1] == KGV_P1 && a.v[0] == KGV_P0);
}
KGV_HD bool fe_equal(const fe& a, const fe& b) {
  fe d;
  fe_sub(d, a, b);
  return fe_is_zero(d);
}

// reduce a 512-bit value t[0..15] modulo p into a weakly reduced element
KGV_HD void fe_reduce_wide(fe& r, const uint32_t* t) {
  // value = lo + hi * 2^256 == lo + hi*977 + (hi << 32).  The multiply-accumulates do the additions for free:
  //   x  = lo + hi_even * 977          (products at even limbs, accumulated straight onto a copy of lo; x[8] = overflow limb)
  //   q  = hi + hi_odd * 977           (the odd-limb products and the "hi << 32" term share the offset of one limb)
  //   x += q << 32                     (the only explicit carry chain of the first fold)
  uint32_t x[9], q[9];
#pragma unroll
  for (int i = 0; i < 8; i++) { x[i] = t[i]; q[i] = t[8 + i]; }
  x[8] = 0; q[8] = 0;
  mad_row4(x, t[8], t[10], t[12], t[14], 977u);
  mad_row4(q, t[9], t[11], t[13], t[15], 977u);
  uint32_t top0 = x[8], top1;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %9;\n\t"
      "addc.cc.u32 %1, %1, %10;\n\t"
      "addc.cc.u32 %2, %2, %11;\n\t"
      "addc.cc.u32 %3, %3, %12;\n\t"
      "addc.cc.u32 %4, %4, %13;\n\t"
      "addc.cc.u32 %5, %5, %14;\n\t"
      "addc.cc.u32 %6, %6, %15;\n\t"
      "addc.cc.u32 %7, %7, %16;\n\t"
      "addc.u32 %8, %17, 0;"
      : "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(top0), "=r"(top1)
      : "r"(q[0]), "r"(q[1]), "r"(q[2]), "r"(q[3]), "r"(q[4]), "r"(q[5]), "r"(q[6]), "r"(q[7]), "r"(q[8]));
#else
  {
    uint64_t c = 0;
    for (int i = 1; i < 8; i++) { c += (uint64_t)x[i] + q[i - 1]; x[i] = (uint32_t)c; c >>= 32; }
    c += (uint64_t)top0 + q[7]; top0 = (uint32_t)c; c >>= 32;
    top1 = q[8] + (uint32_t)c;
  }
#endif
  // second fold: (top1:top0) < 2^34 ; top * C = top*977 + (top << 32)
  uint64_t p977 = (uint64_t)top0 * 977u + ((uint64_t)(top1 * 977u) << 32);
  uint32_t a0 = (uint32_t)p977;
  uint64_t a1w = (p977 >> 32) + top0;
  uint32_t a1 = (uint32_t)a1w;
  uint32_t a2 = top1 + (uint32_t)(a1w >> 32);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = x[i];
  uint32_t c = add8_small3(r.v, a0, a1, a2);
  // c == 1: the sum wrapped past 2^256, so what is left is < (a2:a1:a0) < 2^67 (limbs 3..7 are zero) and the pending
  // 2^256 == 2^32 + 977 fits into limbs 0..2 without further propagation: three unconditional instructions, no branch
  uint32_t k = 977u * c;
#if defined(__CUDACC__)
  asm("add.cc.u32 %0, %0, %3;\n\t"
      "addc.cc.u32 %1, %1, %4;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2])
      : "r"(k), "r"(c));
#else
  {
    uint64_t w = (uint64_t)r.v[0] + k; r.v[0] = (uint32_t)w; w >>= 32;
    w += (uint64_t)r.v[1] + c; r.v[1] = (uint32_t)w; w >>= 32;
    r.v[2] += (uint32_t)w;
  }
#endif
}

// On the device fe_mul / fe_sqr are real (non-inlined) functions taking and returning their
// operands by value: ptxas keeps everything in registers across the call (no stack traffic), and
// the kernels shrink from ~1.4 MB of straight-line SASS to a few tens of KB that stay in the
// instruction cache.  The host unit-test build simply inlines them.
#if defined(__CUDACC__)
static __device__ __noinline__ fe fe_mul_call(fe a, fe b) {
  fe r;
  uint32_t t[16];
  mul_wide(t, a.v, b.v);
  fe_reduce_wide(r, t);
  return r;
}
KGV_HD void fe_mul(fe& r, const fe& a, const fe& b) { r = fe_mul_call(a, b); }
#else
KGV_HD void fe_mul(fe& r, const fe& a, const fe& b) {
  uint32_t t[16];
  mul_wide(t, a.v, b.v);
  fe_reduce_wide(r, t);
}
#endif

// t[0..15] = a^2 : 28 cross products (doubled) + 8 squares = 36 IMAD.WIDE instead of 64.
KGV_HD void sqr_wide(uint32_t* t, const uint32_t* a) {
  // cross products a[i]*a[j], i<j, accumulated with the same even/odd column split as mul_wide
  uint32_t e[18], o[18];
#pragma unroll
  for (int i = 0; i < 18; i++) { e[i] = 0; o[i] = 0; }
  // Each call covers one "row" b = a[i] against the limbs above it, two at a time, by parity.
  // i = 0: j = 1..7
  mad_row4(o + 0, a[1], a[3], a[5], a[7], a[0]);      // odd positions 1,3,5,7 -> o[0,2,4,6]
  mad_row3(e + 2, a[2], a[4], a[6], a[0]);        // even positions 2,4,6
  // i = 1: j = 2..7 ; positions 3..8
  mad_row3(o + 2, a[2], a[4], a[6], a[1]);        // positions 3,5,7 -> o[2,4,6]
  mad_row3(e + 4, a[3], a[5], a[7], a[1]);        // positions 4,6,8
  // i = 2: j = 3..7 ; positions 5..9
  mad_row3(o + 4, a[3], a[5], a[7], a[2]);        // positions 5,7,9 -> o[4,6,8]
  mad_row2(e + 6, a[4], a[6], a[2]);          // positions 6,8
  // i = 3: j = 4..7 ; positions 7..10
  mad_row2(o + 6, a[4], a[6], a[3]);          // positions 7,9 -> o[6,8]
  mad_row2(e + 8, a[5], a[7], a[3]);          // positions 8,10
  // i = 4: j = 5..7 ; positions 9..11
  mad_row2(o + 8, a[5], a[7], a[4]);          // positions 9,11 -> o[8,10]
  mad_row1(e + 10, a[6], a[4]);           // position 10
  // i = 5: j = 6,7 ; positions 11,12
  mad_row1(o + 10, a[6], a[5]);           // position 11 -> o[10]
  mad_row1(e + 12, a[7], a[5]);           // position 12
  // i = 6: j = 7 ; position 13
  mad_row1(o + 12, a[7], a[6]);           // position 13 -> o[12]
  // cross = e + (o << 32); doubled by a funnel shift; diagonal squares added by one IMAD.WIDE chain
  uint32_t x[16];
  merge_eo(x, e, o);
#pragma unroll
  for (int i = 15; i > 0; i--) {
#if defined(__CUDACC__)
    x[i] = __funnelshift_l(x[i - 1], x[i], 1);
#else
    x[i] = (x[i] << 1) | (x[i - 1] >> 31);
#endif
  }
  x[0] <<= 1;
#if defined(__CUDACC__)
  asm("mad.lo.cc.u32  %0, %16, %16, %0;\n\t"
      "madc.hi.cc.u32 %1, %16, %16, %1;\n\t"
      "madc.lo.cc.u32 %2, %17, %17, %2;\n\t"
      "madc.hi.cc.u32 %3, %17, %17, %3;\n\t"
      "madc.lo.cc.u32 %4, %18, %18, %4;\n\t"
      "madc.hi.cc.u32 %5, %18, %18, %5;\n\t"
      "madc.lo.cc.u32 %6, %19, %19, %6;\n\t"
      "madc.hi.cc.u32 %7, %19, %19, %7;\n\t"
      "madc.lo.cc.u32 %8, %20, %20, %8;\n\t"
      "madc.hi.cc.u32 %9, %20, %20, %9;\n\t"
      "madc.lo.cc.u32 %10, %21, %21, %10;\n\t"
      "madc.hi.cc.u32 %11, %21, %21, %11;\n\t"
      "madc.lo.cc.u32 %12, %22, %22, %12;\n\t"
      "madc.hi.cc.u32 %13, %22, %22, %13;\n\t"
      "madc.lo.cc.u32 %14, %23, %23, %14;\n\t"
      "madc.hi.u32    %15, %23, %23, %15;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(x[8]), "+r"(x[9]),
        "+r"(x[10]), "+r"(x[11]), "+r"(x[12]), "+r"(x[13]), "+r"(x[14]), "+r"(x[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]));
#else
  {
    uint64_t c = 0;
    for (int i = 0; i < 8; i++) {
      uint64_t p = (uint64_t)a[i] * a[i];
      uint64_t lo = (uint64_t)x[2 * i] + (uint32_t)p + c;
      x[2 * i] = (uint32_t)lo;
      uint64_t hi = (uint64_t)x[2 * i + 1] + (uint32_t)(p >> 32) + (lo >> 32);
      x[2 * i + 1] = (uint32_t)hi;
      c = hi >> 32;
    }
  }
#endif
#pragma unroll
  for (int i = 0; i < 16; i++) t[i] = x[i];
}

#if defined(__CUDACC__)
static __device__ __noinline__ fe fe_sqr_call(fe a) {
  fe r;
  uint32_t t[16];
  sqr_wide(t, a.v);
  fe_reduce_wide(r, t);
  return r;
}
KGV_HD void fe_sqr(fe& r, const fe& a) { r = fe_sqr_call(a); }
#else
KGV_HD void fe_sqr(fe& r, const fe& a) {
  uint32_t t[16];
  sqr_wide(t, a.v);
  fe_reduce_wide(r, t);
}
#endif

// r = a^(2^n), one fe_sqr call per squaring.  Making a whole run of squarings ONE call instead (the squaring inlined into the loop of a
// non-inlined function, so the exponentiation chains - square root of lift_x, the shared inversion, ~510 squarings per verification - pay the
// by-value call ABI once per run) was measured when the kernels were tuned on the previous target GPU (not re-measured on H100): fewer
// instructions but slower for the field (a second copy of the squaring in the hot code).  The scalar side does use it (sc_pow2k_mul_call,
// kgv_secp.cuh), where it made the scalar inversion of ECDSA faster.
KGV_HD void fe_sqr_n(fe& r, const fe& a, int n) {
  r = a;
  for (int i = 0; i < n; i++) fe_sqr(r, r);
}

// small multiples
KGV_HD void fe_mul3(fe& r, const fe& a) { fe t; fe_add(t, a, a); fe_add(r, t, a); }
// r = 8a: shift left by 3 and fold the three bits that leave the top limb (2^256 == C)
KGV_HD void fe_mul8(fe& r, const fe& a) {
  uint32_t top = a.v[7] >> 29;
  fe t;
#pragma unroll
  for (int i = 7; i > 0; i--) t.v[i] = (a.v[i] << 3) | (a.v[i - 1] >> 29);
  t.v[0] = a.v[0] << 3;
  uint32_t c = add_low2_rare(t.v, 977u * top, top);
  if (c) (void)fe_add_kC(t, 1);
  r = t;
}

// shared prefix of the exponent chains for p-2 and (p+1)/4 (exponent bits from the top: 223 ones, 0, 22 ones, tail)
KGV_HD void fe_pow_x223(fe& x223, fe& x22, fe& x2, const fe& a) {
  fe x3, x6, x9, x11, x44, x88, t;
  fe_sqr(t, a); fe_mul(x2, t, a);
  fe_sqr(t, x2); fe_mul(x3, t, a);
  fe_sqr_n(t, x3, 3); fe_mul(x6, t, x3);
  fe_sqr_n(t, x6, 3); fe_mul(x9, t, x3);
  fe_sqr_n(t, x9, 2); fe_mul(x11, t, x2);
  fe_sqr_n(t, x11, 11); fe_mul(x22, t, x11);
  fe_sqr_n(t, x22, 22); fe_mul(x44, t, x22);
  fe_sqr_n(t, x44, 44); fe_mul(x88, t, x44);
  fe_sqr_n(t, x88, 88); fe_mul(t, t, x88);   // x176
  fe_sqr_n(t, t, 44); fe_mul(t, t, x44);     // x220
  fe_sqr_n(t, t, 3); fe_mul(x223, t, x3);
}
// r = a^(p-2)  (0 -> 0)
KGV_HD void fe_inv(fe& r, const fe& a) {
  fe x223, x22, x2, t;
  fe_pow_x223(x223, x22, x2, a);
  fe_sqr_n(t, x223, 23); fe_mul(t, t, x22);
  fe_sqr_n(t, t, 5); fe_mul(t, t, a);
  fe_sqr_n(t, t, 3); fe_mul(t, t, x2);
  fe_sqr_n(t, t, 2); fe_mul(r, t, a);
}
// r = a^((p+1)/4); true iff r^2 == a
KGV_HD bool fe_sqrt(fe& r, const fe& a) {
  fe x223, x22, x2, t, chk;
  fe_pow_x223(x223, x22, x2, a);
  fe_sqr_n(t, x223, 23); fe_mul(t, t, x22);
  fe_sqr_n(t, t, 6); fe_mul(t, t, x2);
  fe_sqr_n(t, t, 2);
  fe_sqr(chk, t);
  r = t;
  return fe_equal(chk, a);
}

// Big-endian 32-byte strings are handled as 8 numeric words w[0..7], w[0] the most significant
// (the kernels apply bswap32 to the raw little-endian loads once); limbs are little-endian.
KGV_HD uint32_t bswap32(uint32_t x) {
#if defined(__CUDACC__)
  return __byte_perm(x, 0, 0x0123);
#else
  return (x >> 24) | ((x >> 8) & 0xFF00u) | ((x << 8) & 0xFF0000u) | (x << 24);
#endif
}
KGV_HD void limbs_from_be_words(uint32_t* v, const uint32_t* w) {
#pragma unroll
  for (int i = 0; i < 8; i++) v[7 - i] = w[i];
}
// a < b on 8-limb numbers
KGV_HD bool lt8(const uint32_t* a, const uint32_t* b) {
  uint32_t t[8];
  return sub8(t, a, b) != 0;
}

}  // namespace kgv
