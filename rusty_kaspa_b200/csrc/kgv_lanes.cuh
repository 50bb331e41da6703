// kgv_lanes.cuh — secp256k1 field product spread over an eight-lane group, for latency-bound launches.
//
// The per-thread product of kgv_arith.cuh is a chain of ~600 dependent cycles at one warp per scheduler: fine when the
// device is full, the whole cost of a launch that carries a handful of signatures.  Here one field element lives in
// eight consecutive lanes of a warp, lane k of the group holding limb k (the same 8 x 32-bit little-endian limbs, the
// same weak-reduction contract: any representative in [0, 2^256)).  Each lane makes 8 of the 64 limb products, so the
// dependent chain is the product rows of one column plus a few shuffle rounds for the carries.
//
// Masks: every shuffle and vote names the group's own eight lanes, never the full warp, so the four groups of a warp
// may diverge (a group without work leaves as a whole group; the caller keeps each group converged).  Shuffles use
// width 8, so lane indices below are relative to the group.  No local arrays: one limb per lane needs none.
//
// Device-only (shuffles and votes have no host build).  tools/microbench/femul.cu measures the latency of these calls
// next to the per-thread ones; kgv_debug_selftest ops 12 and 13 run them for the tests.  Measured on the H100 at one warp
// per scheduler, a call takes about 1.9x the per-thread product's latency (DESIGN.md §4 K1), so no verify path uses it.
#pragma once
#include <stdint.h>

namespace kgv {

// the group's lane mask and this lane's limb index
struct lane_grp {
  uint32_t mask;
  uint32_t k;
};
__device__ __forceinline__ lane_grp lane_group() {
  const uint32_t lane = threadIdx.x & 31u;
  return lane_grp{0xFFu << (lane & ~7u), lane & 7u};
}

// (x2:x1:x0) += x * y, a 96-bit column accumulator (one IMAD.WIDE pair and a carry into the top word)
__device__ __forceinline__ void lanes_mac(uint32_t& x0, uint32_t& x1, uint32_t& x2, uint32_t x, uint32_t y) {
  asm("mad.lo.cc.u32  %0, %3, %4, %0;\n\t"
      "madc.hi.cc.u32 %1, %3, %4, %1;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(x0), "+r"(x1), "+r"(x2)
      : "r"(x), "r"(y));
}

// Resolve a value held as one limb v and one carry bit g per lane (g of lane k belongs to lane k + 1; lane 7's to
// 2^256) into eight limbs.  A lane whose limb is all ones passes an incoming carry on; the carry into every lane is then
// one 8-bit addition on the group's vote bits (carry-lookahead).  Returns whether the sum wrapped past 2^256; the
// caller folds that.  A lane with g = 1 must not also have v = 0xFFFFFFFF (true for every caller: there v is small).
__device__ __forceinline__ uint32_t lanes_ripple(uint32_t& v, uint32_t g, const lane_grp& grp) {
  const uint32_t sh = __ffs(grp.mask) - 1;
  const uint32_t G = (__ballot_sync(grp.mask, g != 0) >> sh) & 0xFFu;
  const uint32_t X = G | ((__ballot_sync(grp.mask, v == 0xFFFFFFFFu) >> sh) & 0xFFu);
  const uint32_t S = X + G;
  v += ((S ^ X ^ G) >> grp.k) & 1u;  // carry into this lane
  return S >> 8;
}

// r = a * b mod p, weakly reduced; a, b weakly reduced.  Lane k holds limb k of each.
//
// 1. Lane k sums the products a[i] * b[s] with i + s = k (its low column L) and with i + s = k + 8 (its high column
//    H, 2^256 above).  It takes a[(k - s) mod 8] by a rotate shuffle and b[s] by a broadcast; a product goes to L when
//    s <= k and to H otherwise.  L, H < 8 * 2^64.
// 2. 2^256 == C = 2^32 + 977: the high columns fold as z_k = L_k + 977 H_k + H_{k-1} < 2^78 (H_7 = 0, so lane 0's
//    rotated H_{-1} is zero as required).
// 3. The value is sum z_k 2^(32k).  Lane k adds the middle word of z_{k-1} and the top word of z_{k-2}; what rotates
//    past lane 7 sits at 2^256 or 2^288 and is folded by C.  Every lane is then below 2^43.
// 4. One more round passes each lane's word above 32 bits up by one lane (folding lane 7's by C): every lane is below
//    2^33, one limb and a carry bit.
// 5. lanes_ripple.  If the whole sum wrapped past 2^256, what remains is below 2^246 and C is added once more; that
//    cannot wrap again.  The branch is group-uniform (the wrap bit comes from a vote).
__device__ __forceinline__ uint32_t fe_mul_lanes(uint32_t a, uint32_t b, const lane_grp& grp) {
  const uint32_t m = grp.mask, k = grp.k;
  uint32_t l0 = 0, l1 = 0, l2 = 0, h0 = 0, h1 = 0, h2 = 0;
#pragma unroll
  for (uint32_t s = 0; s < 8; s++) {
    const uint32_t x = __shfl_sync(m, a, (k - s) & 7u, 8);
    const uint32_t y = __shfl_sync(m, b, s, 8);
    const uint32_t yl = s <= k ? y : 0u;
    lanes_mac(l0, l1, l2, x, yl);
    lanes_mac(h0, h1, h2, x, y - yl);
  }
  // z = L + 977 H + H_{k-1}
  const uint32_t g0 = __shfl_sync(m, h0, (k - 1) & 7u, 8), g1 = __shfl_sync(m, h1, (k - 1) & 7u, 8),
                 g2 = __shfl_sync(m, h2, (k - 1) & 7u, 8);
  uint32_t over = 0;  // stays 0: z < 2^78
  lanes_mac(l0, l1, l2, h0, 977u);
  lanes_mac(l1, l2, over, h1, 977u);
  l2 += h2 * 977u;
  asm("add.cc.u32 %0, %0, %3;\n\t"
      "addc.cc.u32 %1, %1, %4;\n\t"
      "addc.u32 %2, %2, %5;"
      : "+r"(l0), "+r"(l1), "+r"(l2)
      : "r"(g0), "r"(g1), "r"(g2));
  // step 3: lane 0 receives z1_7 and z2_6 (both at 2^256), lane 1 z2_7 (at 2^288 == 977 * 2^32 + 2^64)
  const uint32_t r1 = __shfl_sync(m, l1, (k - 1) & 7u, 8), r2 = __shfl_sync(m, l2, (k - 2) & 7u, 8);
  const uint32_t w17 = __shfl_sync(m, l1, 7, 8), w26 = __shfl_sync(m, l2, 6, 8), w27 = __shfl_sync(m, l2, 7, 8);
  uint64_t x = (uint64_t)l0 + (uint64_t)(k >= 1 ? 1u : 977u) * r1 + (uint64_t)(k >= 2 ? 1u : 977u) * r2;
  x += k == 1 ? (uint64_t)w17 + w26 : k == 2 ? (uint64_t)w27 : 0u;
  // step 4
  const uint32_t xh = (uint32_t)(x >> 32);
  const uint32_t q = __shfl_sync(m, xh, (k - 1) & 7u, 8), q7 = __shfl_sync(m, xh, 7, 8);
  uint64_t y = (uint64_t)(uint32_t)x + (uint64_t)(k == 0 ? 977u : 1u) * q + (k == 1 ? q7 : 0u);
  uint32_t v = (uint32_t)y;
  if (lanes_ripple(v, (uint32_t)(y >> 32), grp)) {
    y = (uint64_t)v + (k == 0 ? 977u : k == 1 ? 1u : 0u);
    v = (uint32_t)y;
    (void)lanes_ripple(v, (uint32_t)(y >> 32), grp);
  }
  return v;
}

// r = a^2 mod p.  Each lane makes eight products whether or not the operands are equal, and the chain after them is the
// product's, so a squaring costs what a product costs (femul.cu measures both).
__device__ __forceinline__ uint32_t fe_sqr_lanes(uint32_t a, const lane_grp& grp) { return fe_mul_lanes(a, a, grp); }

}  // namespace kgv
