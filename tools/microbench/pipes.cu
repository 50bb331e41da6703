// Integer / FP64 pipe throughput probe (build with the -gencode flags of __graft_entry__.py).
// Measures per-SM lane-ops/clk for the instruction mixes a 256-bit modular
// multiply is made of, so DESIGN.md's IMAD roofline is a measured number.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITERS 4096
#define ILP 8

template <int MODE>
__global__ void __launch_bounds__(256) probe(uint32_t* out, uint32_t seed, unsigned long long* cycles) {
  uint32_t a[ILP], b[ILP];
  uint64_t w[ILP];
  double d[ILP];
  uint32_t x = seed + threadIdx.x, y = seed * 3u + 7u;
#pragma unroll
  for (int i = 0; i < ILP; i++) { a[i] = x + i; b[i] = y ^ i; w[i] = (uint64_t)x * (i + 1); d[i] = (double)(x + i); }
  double dm = (double)y * 1e-9, da = 0.5;
  unsigned long long t0 = clock64();
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < ILP; i++) {
      if (MODE == 0) {  // IMAD 32-bit lo
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(y), "r"(b[i]));
      } else if (MODE == 1) {  // IMAD.WIDE.U32
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(y));
      } else if (MODE == 2) {  // IMAD.HI
        asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(y), "r"(b[i]));
      } else if (MODE == 3) {  // IADD3
        asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b[i]));
      } else if (MODE == 4) {  // DFMA
        asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(dm), "d"(da));
      } else if (MODE == 5) {  // IMAD.WIDE + IADD3 interleaved 1:1
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(y));
        asm volatile("add.u32 %0, %0, %1;" : "+r"(b[i]) : "r"(x));
      } else if (MODE == 6) {  // IMAD.WIDE + DFMA interleaved 1:1
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(y));
        asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(dm), "d"(da));
      } else if (MODE == 7) {  // carry chain: mad.lo.cc / madc.hi.cc pairs (what a limb product row is)
        asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.cc.u32 %1, %2, %3, %1;\n\taddc.u32 %1, %1, 0;"
                     : "+r"(a[i]), "+r"(b[i]) : "r"(x), "r"(y));
      } else if (MODE == 8) {  // IMAD + IADD3 1:1
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(y), "r"(x));
        asm volatile("add.u32 %0, %0, %1;" : "+r"(b[i]) : "r"(x));
      } else if (MODE == 10) {  // IMAD.WIDE, all operands distinct registers (no operand reuse)
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(b[i]));
      } else if (MODE == 11) {  // same through C++ (lets ptxas pick the form)
        w[i] += (uint64_t)a[i] * b[i];
      } else if (MODE == 12) {  // 32-bit IMAD, distinct operands
        asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b[i]), "r"(b[(i + 1) % ILP]));
      } else if (MODE == 13) {  // IMAD.WIDE distinct, accumulator chain of length 2 (two products per accumulator per pass)
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i / 2]) : "r"(a[i]), "r"(b[i]));
      } else if (MODE == 14) {  // product without addend + xor consume (IMAD.WIDE RZ + 2 LOP3)
        uint64_t t;
        asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(t) : "r"(a[i]), "r"(b[i]));
        w[i] ^= t;
      } else if (MODE == 15) {  // IMAD.WIDE accumulate, multiplicand = own low word (nothing loop-invariant)
        asm volatile("{\n\t.reg .b32 lo, hi;\n\tmov.b64 {lo, hi}, %0;\n\tmad.wide.u32 %0, lo, %1, %0;\n\t}" : "+l"(w[i]) : "r"(b[i]));
      } else if (MODE == 16) {  // IMAD.WIDE without addend, multiplicand = own low word
        asm volatile("{\n\t.reg .b32 lo, hi;\n\tmov.b64 {lo, hi}, %0;\n\tmul.wide.u32 %0, lo, %1;\n\t}" : "+l"(w[i]) : "r"(b[i]));
      } else if (MODE == 17) {  // carry form: (hi:lo) = lo * b + (hi:lo) via mad.lo.cc / madc.hi (one IMAD.WIDE.U32 with carry out... )
        asm volatile("{\n\t.reg .b32 lo, hi, t;\n\tmov.b64 {lo, hi}, %0;\n\tmov.b32 t, lo;\n\tmad.lo.cc.u32 lo, t, %1, lo;\n\tmadc.hi.u32 hi, t, %1, hi;\n\tmov.b64 %0, {lo, hi};\n\t}" : "+l"(w[i]) : "r"(b[i]));
      } else if (MODE == 18) {  // 32-bit IMAD, multiplicand = own value, distinct operands
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(b[(i + 3) % ILP]));
      } else if (MODE == 9) {  // IMAD.WIDE with carry-in/out chain via add.cc on 64-bit halves
        asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(y));
        asm volatile("add.cc.u32 %0, %0, %1;\n\taddc.u32 %0, %0, %1;" : "+r"(b[i]) : "r"(x));
      }
    }
  }
  unsigned long long t1 = clock64();
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < ILP; i++) acc ^= a[i] ^ b[i] ^ (uint32_t)w[i] ^ (uint32_t)(w[i] >> 32) ^ (uint32_t)__double_as_longlong(d[i]);
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int MODE>
void run(const char* name, int ops_per_iter, int nsm, uint32_t* out, unsigned long long* cyc) {
  int blocks = nsm * 4;  // 4 x 256 threads = 32 warps/SM
  probe<MODE><<<blocks, 256>>>(out, 12345u, cyc);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  probe<MODE><<<blocks, 256>>>(out, 12345u, cyc);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  unsigned long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
  double lane_ops = (double)blocks * 256 * ITERS * ILP * ops_per_iter;
  printf("%-34s %8.3f ms  %10llu cyc(block0)  %7.2f lane-ops/clk/SM (by clock64)  %8.2f Gops/s\n", name, ms, c,
         (double)4 * 256 * ITERS * ILP * ops_per_iter / (double)c, lane_ops / ms * 1e-6);
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  printf("device %s SMs=%d clock=%d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  uint32_t* out; unsigned long long* cyc;
  cudaMalloc(&out, (size_t)p.multiProcessorCount * 4 * 256 * 4); cudaMalloc(&cyc, 8);
  int n = p.multiProcessorCount;
  run<0>("IMAD (mad.lo.u32)", 1, n, out, cyc);
  run<1>("IMAD.WIDE.U32", 1, n, out, cyc);
  run<2>("IMAD.HI", 1, n, out, cyc);
  run<3>("IADD3 (add.u32)", 1, n, out, cyc);
  run<4>("DFMA", 1, n, out, cyc);
  run<5>("IMAD.WIDE + IADD 1:1", 2, n, out, cyc);
  run<6>("IMAD.WIDE + DFMA 1:1", 2, n, out, cyc);
  run<7>("mad.lo.cc/madc.hi.cc/addc", 3, n, out, cyc);
  run<8>("IMAD + IADD 1:1", 2, n, out, cyc);
  run<9>("IMAD.WIDE + 2x IADD.cc", 3, n, out, cyc);
  run<10>("IMAD.WIDE distinct operands", 1, n, out, cyc);
  run<11>("IMAD.WIDE distinct (C++)", 1, n, out, cyc);
  run<12>("IMAD distinct operands", 1, n, out, cyc);
  run<13>("IMAD.WIDE distinct, chain 2", 1, n, out, cyc);
  run<14>("mul.wide + xor.b64", 1, n, out, cyc);
  run<15>("IMAD.WIDE acc, dependent operand", 1, n, out, cyc);
  run<16>("IMAD.WIDE RZ, dependent operand", 1, n, out, cyc);
  run<17>("mad.lo.cc+madc.hi dependent", 1, n, out, cyc);
  run<18>("IMAD dependent operand", 1, n, out, cyc);
  return 0;
}
