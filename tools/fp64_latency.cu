// Microbenchmark: dependent-issue latencies (cycles) of the FP64 / shuffle / shared-memory / DMMA instructions that sit on the
// solver's pivot and back-substitution recurrences; the dependent latency and one-warp issue interval of every FP64 MMA shape
// (fp64_mma.cuh); whether one m16n8k4 gives the same bits as the two m8n8k4 of its row blocks.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_latency fp64_latency.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "fp64_mma.cuh"
#define N 4096
__global__ void k(double* out, long long* cyc, double seed) {
  __shared__ double sm[64];
  sm[threadIdx.x & 63] = seed;
  __syncthreads();
  double x = seed + threadIdx.x * 1e-9, y = 1.0000001 + seed * 1e-12, keep = 0;
  long long t0, t1;
  // DFMA chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = fma(x, y, 1e-9);
  t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0; keep += x;
  // DMUL chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = x * y;
  t1 = clock64(); if (threadIdx.x == 0) cyc[1] = t1 - t0; keep += x;
  // DADD chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = x + y;
  t1 = clock64(); if (threadIdx.x == 0) cyc[2] = t1 - t0; keep += x;
  // reciprocal chain 1/x
  x = 1.5 + threadIdx.x * 1e-9 + keep * 1e-300;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) x = 1.0 / x + 0.25;
  t1 = clock64(); if (threadIdx.x == 0) cyc[3] = t1 - t0; keep += x;
  // shuffle (64-bit) chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31);
  t1 = clock64(); if (threadIdx.x == 0) cyc[4] = t1 - t0; keep += x;
  // shared-memory load chain (pointer chasing through an index held in the value)
  int idx = threadIdx.x & 63;
  sm[idx] = (double)((idx + 1) & 63);
  __syncthreads();
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) idx = (int)sm[idx];
  t1 = clock64(); if (threadIdx.x == 0) cyc[5] = t1 - t0;
  // sqrt + sincos chains
  x = 1.5 + keep * 1e-300;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) x = sqrt(x) + 1.0;
  t1 = clock64(); if (threadIdx.x == 0) cyc[6] = t1 - t0; keep += x;
  x = 0.3 + keep * 1e-300;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) { double s, c; sincos(x, &s, &c); x = s * 0.5 + c * 0.1; }
  t1 = clock64(); if (threadIdx.x == 0) cyc[7] = t1 - t0; keep += x;
  // __syncthreads cost is measured in the other kernel
  double acc = x + idx + keep;
  out[threadIdx.x] = acc;
}
// Per FP64 MMA shape: cyc[0] a dependent chain (each MMA accumulates into the previous one's result), cyc[1] N MMAs over 8
// independent accumulators (the issue interval of one warp).
template <Shape S>
__global__ void kmma(double* out, long long* cyc) {
  constexpr int ACC = Mma<S>::ACC;
  double c[ACC] = {}, d[8 * ACC] = {}, a = 1e-3, b = 1e-3;
  long long t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) Mma<S>::run(c, a, b);
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0;
  t0 = clock64();
  for (int i = 0; i < N / 8; ++i) {
#pragma unroll
    for (int q = 0; q < 8; ++q) Mma<S>::run(d + ACC * q, a, b);
  }
  t1 = clock64(); if (threadIdx.x == 0) cyc[1] = t1 - t0;
  double acc = 0;
  for (int i = 0; i < ACC; ++i) acc += c[i];
  for (int i = 0; i < 8 * ACC; ++i) acc += d[i];
  out[threadIdx.x] = acc;
}
template <Shape S>
void mma_rows(double* out, long long* cyc) {
  long long h[2];
  kmma<S><<<1, 32>>>(out, cyc); cudaDeviceSynchronize();
  cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
  printf("DMMA %-9s dependent          %8.1f cycles/op\n", Mma<S>::name, (double)h[0] / N);
  printf("DMMA %-9s issue (8 indep)    %8.1f cycles/op\n", Mma<S>::name, (double)h[1] / N);
}
// m16n8k4 against two m8n8k4 on the same operands (A rows g / g + 8, one B), 256 chained k-steps of random operands per lane: counts
// the accumulator values whose bits differ.
__device__ double rnd(unsigned long long& s) { s = s * 6364136223846793005ull + 1442695040888963407ull; return ((s >> 11) * 0x1.0p-53 - 0.5) * ((s & 7) + 1); }
__global__ void kbits(unsigned long long* nbad) {
  unsigned long long s = 1234567ull + 7919ull * (blockIdx.x * 32 + threadIdx.x);
  double w[4] = {}, n0[2] = {}, n1[2] = {};
  for (int it = 0; it < 256; ++it) {
    const double a0 = rnd(s), a1 = rnd(s), b = rnd(s);
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};" : "+d"(w[0]), "+d"(w[1]), "+d"(w[2]), "+d"(w[3]) : "d"(a0), "d"(a1), "d"(b));
    Mma<M8N8K4>::run(n0, a0, b);
    Mma<M8N8K4>::run(n1, a1, b);
  }
  const double ref[4] = {n0[0], n0[1], n1[0], n1[1]};
  for (int i = 0; i < 4; ++i) if (__double_as_longlong(w[i]) != __double_as_longlong(ref[i])) atomicAdd(nbad, 1ull);
}
__global__ void kbar(long long* cyc) {
  long long t0 = clock64();
  for (int i = 0; i < 1024; ++i) __syncthreads();
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
int main() {
  double* out; long long* cyc; cudaMalloc(&out, 1024 * 8); cudaMalloc(&cyc, 16 * 8);
  long long h[16];
  const char* names[] = {"DFMA", "DMUL", "DADD", "1.0/x (+DADD)", "SHFL.64", "LDS chase (+cvt)", "sqrt (+DADD)", "sincos (+2 DMUL,DADD)"};
  for (int warps = 1; warps <= 1; ++warps) {
    k<<<1, 32 * warps>>>(out, cyc, 1.0); cudaDeviceSynchronize();
    cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
    for (int i = 0; i < 8; ++i) printf("%-32s %8.1f cycles/op\n", names[i], (double)h[i] / N);
  }
  mma_rows<M8N8K4>(out, cyc);
  mma_rows<M16N8K4>(out, cyc);
  mma_rows<M16N8K8>(out, cyc);
  mma_rows<M16N8K16>(out, cyc);
  {
    unsigned long long* nbad; cudaMalloc(&nbad, 8); cudaMemset(nbad, 0, 8);
    kbits<<<1024, 32>>>(nbad); cudaDeviceSynchronize();
    unsigned long long n; cudaMemcpy(&n, nbad, 8, cudaMemcpyDeviceToHost); cudaFree(nbad);
    printf("m16n8k4 vs 2 x m8n8k4: %llu of %d accumulator values differ in any bit\n", n, 1024 * 32 * 4);
  }
  for (int thr : {64, 256, 512, 1024}) { kbar<<<1, thr>>>(cyc); cudaDeviceSynchronize(); cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost); printf("__syncthreads %4d threads      %8.1f cycles\n", thr, (double)h[0] / 1024); }
  printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
