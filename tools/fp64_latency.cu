// Microbenchmark: dependent-issue latencies (cycles) of the FP64 / shuffle / shared-memory / DMMA instructions that sit on the
// solver's pivot and back-substitution recurrences.  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_latency fp64_latency.cu
#include <cstdio>
#include <cuda_runtime.h>
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
  // DMMA m8n8k4 dependent chain
  double c0 = 0, c1 = 0, a = 1e-3, b = 1e-3;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
  t1 = clock64(); if (threadIdx.x == 0) cyc[6] = t1 - t0;
  // DMMA throughput: 8 independent accumulators
  double d[16]; for (int i = 0; i < 16; ++i) d[i] = 0;
  t0 = clock64();
  for (int i = 0; i < N / 8; ++i) {
#pragma unroll
    for (int q = 0; q < 8; ++q) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d[2 * q]), "+d"(d[2 * q + 1]) : "d"(a), "d"(b));
  }
  t1 = clock64(); if (threadIdx.x == 0) cyc[7] = t1 - t0;
  // sqrt + sincos chains
  x = 1.5 + keep * 1e-300;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) x = sqrt(x) + 1.0;
  t1 = clock64(); if (threadIdx.x == 0) cyc[8] = t1 - t0; keep += x;
  x = 0.3 + keep * 1e-300;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) { double s, c; sincos(x, &s, &c); x = s * 0.5 + c * 0.1; }
  t1 = clock64(); if (threadIdx.x == 0) cyc[9] = t1 - t0; keep += x;
  // __syncthreads cost is measured in the other kernel
  double acc = x + c0 + c1 + idx + keep; for (int i = 0; i < 16; ++i) acc += d[i];
  out[threadIdx.x] = acc;
}
__global__ void kbar(long long* cyc) {
  long long t0 = clock64();
  for (int i = 0; i < 1024; ++i) __syncthreads();
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
int main() {
  double* out; long long* cyc; cudaMalloc(&out, 1024 * 8); cudaMalloc(&cyc, 16 * 8);
  long long h[16];
  const char* names[] = {"DFMA", "DMUL", "DADD", "1.0/x (+DADD)", "SHFL.64", "LDS chase (+cvt)", "DMMA m8n8k4 dependent", "DMMA m8n8k4 issue (8 indep)", "sqrt (+DADD)", "sincos (+2 DMUL,DADD)"};
  for (int warps = 1; warps <= 1; ++warps) {
    k<<<1, 32 * warps>>>(out, cyc, 1.0); cudaDeviceSynchronize();
    cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
    for (int i = 0; i < 10; ++i) printf("%-32s %8.1f cycles/op\n", names[i], (double)h[i] / (i == 7 ? N : N));
  }
  for (int thr : {64, 256, 512, 1024}) { kbar<<<1, thr>>>(cyc); cudaDeviceSynchronize(); cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost); printf("__syncthreads %4d threads      %8.1f cycles\n", thr, (double)h[0] / 1024); }
  printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
