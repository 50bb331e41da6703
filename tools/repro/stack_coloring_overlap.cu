// Reproducer (nvcc 12.9, found when building for sm_100a) for the miscompile first seen as "results are wrong when the multiplications are inlined"
// (DESIGN.md §6).  Root cause: two local arrays that are live at the same time get the SAME stack offset.
// Here: `uint32_t r[96]` (written by u3072_canonical, read in the loop after the hasher is initialised) and the
// 14-byte key string inside the inlined keyed-BLAKE2b init (KEY_ARRAY=1).  The kernel then outputs the ASCII key
// "MuHashFinalize" instead of the number 1:   r[0..3] = 6148754d 69466873 696c616e 0000657a.
// Visible in the PTX: `add.u64 %rdA, %SPL, 0` for r[] and `add.u64 %rdB, %SPL, 0` for the key bytes.
// It does not depend on ptxas (-Xptxas -O0 fails too), on the number of inlined multiplier call sites (SITES=1 fails),
// or on how the block multiplier is called; it disappears when the multiplier is a __noinline__ function (different
// stack layout) or when the key array is removed (KEY_ARRAY=0, the shipped form: key given as two 64-bit words).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DKEY_ARRAY=1 -o repro_bad  stack_coloring_overlap.cu
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DKEY_ARRAY=0 -o repro_good stack_coloring_overlap.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../rusty_kaspa_b200/csrc/kgv_muhash.cuh"
using namespace kgv;
#ifndef SITES
#define SITES 1
#endif
#ifndef TAIL
#define TAIL 2
#endif
#ifndef KEY_ARRAY
#define KEY_ARRAY 1
#endif
// the form the library used when the problem was found: key bytes in a local array, absorbed byte by byte
__device__ __forceinline__ void init_finalize_with_key_array(Blake2b& h) {
  const char dom[14] = {'M', 'u', 'H', 'a', 's', 'h', 'F', 'i', 'n', 'a', 'l', 'i', 'z', 'e'};
  b2b_init(h, B2B_UNKEYED);
  h.h[0] = kB2bIV[0] ^ (0x01010000ull ^ (14ull << 8) ^ 32ull);
  for (uint32_t b = 0; b < 128; b++) b2b_byte(h, b < 14 ? (uint32_t)(uint8_t)dom[b] : 0u);
}
__device__ __forceinline__ void coop_mul(U3072Coop* sm, int lane, bool act, uint32_t* r, const uint32_t* a, const uint32_t* b) {
  u3072_coop_mul_mod(*sm, lane, act, r, 1, 0, a, 1, 0, b, 1, 0);
}
__global__ void k_sites(uint32_t* w, uint32_t* out, int n) {
  __shared__ U3072Coop sm;
  const int lane = threadIdx.x & 15;
  const bool act = threadIdx.x < 16;
  uint32_t *den = w, *cur = w + 96;
  if (act) for (int i = lane; i < 96; i += 16) cur[i] = den[i];
  __syncwarp();
  for (int q = 0; q < n; q++) {
    coop_mul(&sm, lane, act, cur, cur, cur);
#if SITES >= 2
    coop_mul(&sm, lane, act, cur, cur, den);
#endif
#if SITES >= 3
    coop_mul(&sm, lane, act, cur, den, cur);
#endif
#if SITES >= 4
    coop_mul(&sm, lane, act, cur, cur, cur);
#endif
  }
  if (threadIdx.x == 0) {
    uint32_t r[96];
    u3072_canonical(r, cur, 1, 0);
#if TAIL == 2
    Blake2b h;
#if KEY_ARRAY
    init_finalize_with_key_array(h);
#else
    b2b_init_muhash_finalize(h);
#endif
    for (int i = 0; i < 96; i++) { out[i] = r[i]; b2b_u32(h, r[i]); }
    uint64_t d[4];
    b2b_final(h, d);
    for (int i = 0; i < 4; i++) { out[96 + 2 * i] = (uint32_t)d[i]; out[96 + 2 * i + 1] = (uint32_t)(d[i] >> 32); }
#else
    for (int i = 0; i < 96; i++) out[i] = r[i];
#endif
  }
}
int main() {
  uint32_t *w, *o;
  cudaMalloc(&w, 4096); cudaMalloc(&o, 512);
  for (int n : {1, 3}) {
    uint32_t h[96] = {1};
    cudaMemset(w, 0, 4096);
    cudaMemcpy(w, h, sizeof h, cudaMemcpyHostToDevice);
    k_sites<<<1, 32>>>(w, o, n);
    uint32_t r[96];
    cudaError_t e = cudaMemcpy(r, o, sizeof r, cudaMemcpyDeviceToHost);
    bool one = r[0] == 1;
    for (int i = 1; i < 96; i++) one = one && r[i] == 0;
    printf("KEY_ARRAY=%d SITES=%d TAIL=%d n=%d -> 1 stays 1 ? %s (%s)  r[0..3]=%08x %08x %08x %08x\n", KEY_ARRAY, SITES, TAIL, n, one ? "yes" : "NO", cudaGetErrorString(e), r[0], r[1], r[2], r[3]);
  }
  return 0;
}
