// Latency/throughput probe of the field multiply and square subroutines (the exact code the verify kernels
// call) as a function of resident warps per SM sub-partition: a chain of dependent fe_mul / fe_sqr per thread,
// one block per SM with 128*W threads.  Prints cycles per call per warp and calls/clk/SM.
// The lane modes run the eight-lane product of kgv_lanes.cuh: each group of eight lanes carries one dependent chain, so
// at one warp per scheduler "cycles per call per warp" is the latency of one cooperative call.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../rusty_kaspa_b200/csrc/kgv_arith.cuh"
#include "../../rusty_kaspa_b200/csrc/kgv_lanes.cuh"
using namespace kgv;

template <int MODE>
__global__ void probe(uint32_t* out, int iters) {
  fe a, b;
  const lane_grp g = lane_group();
  for (int i = 0; i < 8; i++) { a.v[i] = 0x9E3779B9u * (threadIdx.x + 1 + i) + blockIdx.x; b.v[i] = 0x85EBCA6Bu * (threadIdx.x + 7 + i); }
#pragma unroll 1
  for (int it = 0; it < iters; it++) {
    if (MODE == 0) fe_mul(a, a, b);
    else if (MODE == 1) fe_sqr(a, a);
    else if (MODE == 2) { fe_mul(a, a, b); fe_sqr(b, b); }          // two independent chains
    else if (MODE == 3) { fe_add(a, a, b); }
    else if (MODE == 4) { fe_sub(a, a, b); }
    else if (MODE == 5) { a.v[0] = fe_mul_lanes(a.v[0], b.v[0], g); }
    else if (MODE == 6) { a.v[0] = fe_sqr_lanes(a.v[0], g); }
  }
  uint32_t acc = 0;
  for (int i = 0; i < 8; i++) acc ^= a.v[i] ^ b.v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int MODE>
void run(const char* name, int calls_per_iter, int nsm, uint32_t* out, double ghz) {
  for (int w = 1; w <= 8; w++) {
    int threads = 128 * w, iters = 20000;
    probe<MODE><<<nsm, threads>>>(out, 100);
    cudaDeviceSynchronize();
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    probe<MODE><<<nsm, threads>>>(out, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double cyc = ms * 1e-3 * ghz * 1e9;
    printf("%-22s warps/SMSP %d  %8.3f ms  %7.1f cycles per call per warp  %6.1f scheduler-cycles per call\n", name, w, ms,
           cyc / (iters * calls_per_iter), cyc / (iters * calls_per_iter) / w);
  }
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  double ghz = khz * 1e-6;
  printf("device %s SMs=%d clock=%.3f GHz\n", p.name, p.multiProcessorCount, ghz);
  uint32_t* out; cudaMalloc(&out, (size_t)p.multiProcessorCount * 1024 * 4);
  run<0>("fe_mul chain", 1, p.multiProcessorCount, out, ghz);
  run<1>("fe_sqr chain", 1, p.multiProcessorCount, out, ghz);
  run<2>("fe_mul + fe_sqr indep", 2, p.multiProcessorCount, out, ghz);
  run<3>("fe_add chain", 1, p.multiProcessorCount, out, ghz);
  run<4>("fe_sub chain", 1, p.multiProcessorCount, out, ghz);
  run<5>("fe_mul_lanes chain", 1, p.multiProcessorCount, out, ghz);
  run<6>("fe_sqr_lanes chain", 1, p.multiProcessorCount, out, ghz);
  return 0;
}
