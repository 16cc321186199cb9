// fpmul_probe.cu -- what the 381-bit Montgomery product of fp.cuh sustains when nothing else is in the way (operands in
// registers, no memory traffic, loop body small enough for the instruction cache): the practical ceiling for the MSM
// bucket-accumulate kernel.  Variants: CHAINS independent dependency chains per thread, inlined vs out-of-line product.
//   build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I kyber_b200/csrc -I tools/probe -o tools/probe/fpmul_probe tools/probe/fpmul_probe.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "fp.cuh"
#include "fp_kara.cuh"
#include "fp29.cuh"
#include "constants.cuh"
using namespace b2k;
using F = Fp<Bls381Fp>;

// FORM 0: CIOS product (fp_mul), 1: Karatsuba wide product + redc_wide (fp_kara.cuh: fp_mul_k_inl),
//      2: sum of two products with one reduction (fp_kara.cuh: fp_mul_sum2_inl; counted as two products)
template <int CHAINS, bool NOINLINE, int FORM = 0>
__global__ void __launch_bounds__(128) k_mul(int iters, uint32_t* out, uint32_t seed) {
  F a[CHAINS], b;
#pragma unroll
  for (int c = 0; c < CHAINS; c++)
#pragma unroll
    for (int j = 0; j < 12; j++) a[c].v[j] = seed * (c + 3) + j + threadIdx.x;
#pragma unroll
  for (int j = 0; j < 12; j++) b.v[j] = seed + 7 * j + blockIdx.x;
  a[0].v[11] &= 0x0fffffffu; b.v[11] &= 0x0fffffffu;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CHAINS; c++) {
      if (FORM == 1) fp_mul_k_inl(a[c], a[c], b);
      else if (FORM == 2) fp_mul_sum2_inl(a[c], a[c], b, b, a[c]);
      else if (NOINLINE) fp_mul_c(a[c], a[c], b);
      else fp_mul(a[c], a[c], b);
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; c++)
#pragma unroll
    for (int j = 0; j < 12; j++) s ^= a[c].v[j];
  if (s == 0x12345) out[0] = s;
}

using G = Fp29<Bls381Fp29>;
// MODE 0: products, 1: squarings, 2: product + lazy sub + add per step (the mix of a group addition)
template <int CHAINS, int MODE>
__global__ void __launch_bounds__(128) k_mul29(int iters, uint32_t* out, uint32_t seed) {
  G a[CHAINS], b;
#pragma unroll
  for (int c = 0; c < CHAINS; c++)
#pragma unroll
    for (int j = 0; j < 14; j++) a[c].v[j] = (seed * (c + 3) + j + threadIdx.x) & M29;
#pragma unroll
  for (int j = 0; j < 14; j++) b.v[j] = (seed + 7 * j + blockIdx.x) & M29;
  for (int c = 0; c < CHAINS; c++) a[c].v[13] &= 15u;
  b.v[13] &= 15u;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < CHAINS; c++) {
      if (MODE == 0) fp29_mul(a[c], a[c], b);
      else if (MODE == 1) fp29_sqr(a[c], a[c]);
      else { G t; fp29_mul(t, a[c], b); fp29_sub(t, t, b); fp29_add(a[c], t, b); fp29_mul(a[c], a[c], t); }
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; c++)
#pragma unroll
    for (int j = 0; j < 14; j++) s ^= a[c].v[j];
  if (s == 0x12345) out[0] = s;
}

template <int CHAINS, int MODE>
static void run29(const char* name, int blocks_per_sm, int sms, int clk_khz, uint32_t* out) {
  const int iters = 2048;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  k_mul29<CHAINS, MODE><<<sms * blocks_per_sm, 128>>>(64, out, 5);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k_mul29<CHAINS, MODE><<<sms * blocks_per_sm, 128>>>(iters, out, 9);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  const double muls = (double)sms * blocks_per_sm * 128 * iters * CHAINS * (MODE == 2 ? 2 : 1);
  printf("%-28s blocks/SM %d  %8.3f ms  %.3e products/s\n", name, blocks_per_sm, ms, muls / (ms * 1e-3));
  (void)clk_khz;
}

template <int CHAINS, bool NI, int FORM = 0>
static void run(const char* name, int blocks_per_sm, int sms, int clk_khz, uint32_t* out) {
  const int iters = 2048;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  k_mul<CHAINS, NI, FORM><<<sms * blocks_per_sm, 128>>>(64, out, 5);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k_mul<CHAINS, NI, FORM><<<sms * blocks_per_sm, 128>>>(iters, out, 9);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  const double muls = (double)sms * blocks_per_sm * 128 * iters * CHAINS * (FORM == 2 ? 2 : 1);
  const double per_s = muls / (ms * 1e-3);
  const double imad_clk_sm = muls * 302.0 / (ms * 1e-3 * clk_khz * 1e3) / sms;
  printf("%-28s blocks/SM %d  %8.3f ms  %.3e fp_mul/s  %5.1f IMAD-class thread-instr/clk/SM\n", name, blocks_per_sm, ms, per_s, imad_clk_sm);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  int clk = 0;
  cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  uint32_t* out;
  cudaMalloc(&out, 8);
  const int sms = p.multiProcessorCount;
  printf("%s, %d SMs, max SM clock %d MHz\n", p.name, sms, clk / 1000);
  for (int bps : {2, 4, 8}) {
    run<1, false, 1>("karatsuba, 1 chain", bps, sms, clk, out);
    run<2, false, 1>("karatsuba, 2 chains", bps, sms, clk, out);
    run<1, false, 2>("sum of two, 1 chain", bps, sms, clk, out);
    run<2, false, 2>("sum of two, 2 chains", bps, sms, clk, out);
    run<1, false>("inline, 1 chain", bps, sms, clk, out);
    run<2, false>("inline, 2 chains", bps, sms, clk, out);
    run<4, false>("inline, 4 chains", bps, sms, clk, out);
    run<1, true>("out-of-line, 1 chain", bps, sms, clk, out);
    run<4, true>("out-of-line, 4 chains", bps, sms, clk, out);
    run29<1, 0>("radix-29 mul, 1 chain", bps, sms, clk, out);
    run29<2, 0>("radix-29 mul, 2 chains", bps, sms, clk, out);
    run29<1, 1>("radix-29 sqr, 1 chain", bps, sms, clk, out);
    run29<1, 2>("radix-29 mul+sub+add mix", bps, sms, clk, out);
  }
  return 0;
}
