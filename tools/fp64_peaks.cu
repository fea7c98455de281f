// Microbenchmark: measured FP64 throughput ceilings of one GPU -- the denominators of a second roofline of the residual / solver
// kernels next to the data-sheet figures bench.py divides by:
//   * DFMA (SIMT FP64 pipe): every thread runs 8 independent FMA chains;
//   * DMMA (mma.sync.m8n8k4.f64, the FP64 tensor shape the kernels use): every warp runs 8 / 21
//     independent accumulator fragments (21 = the vision tile's upper block triangle);
//   * both together (alternating warps), to see whether the two pipes overlap.
// Timed with CUDA events over a grid that fills all SMs (SM count x 8 CTAs x 256 threads), best of 5.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peaks fp64_peaks.cu && ./fp64_peaks > fp64_peaks.json
#include <cstdio>
#include <cuda_runtime.h>

constexpr int ITERS = 4096;

__global__ void dfma_kernel(double* out, double seed) {
  double x[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) x[q] = seed + 1e-9 * (threadIdx.x + q);
  const double y = 1.0000001 + seed * 1e-12;
  for (int i = 0; i < ITERS; ++i) {
#pragma unroll
    for (int q = 0; q < 8; ++q) x[q] = fma(x[q], y, 1e-9);
  }
  double s = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) s += x[q];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NACC>
__global__ void dmma_kernel(double* out, double seed) {
  double d[2 * NACC];
#pragma unroll
  for (int q = 0; q < 2 * NACC; ++q) d[q] = 0.0;
  const double a = 1e-3 + seed * 1e-9 * threadIdx.x, b = 1e-3;
  for (int i = 0; i < ITERS; ++i) {
#pragma unroll
    for (int q = 0; q < NACC; ++q) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d[2 * q]), "+d"(d[2 * q + 1]) : "d"(a), "d"(b));
  }
  double s = 0;
#pragma unroll
  for (int q = 0; q < 2 * NACC; ++q) s += d[q];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void mixed_kernel(double* out, double seed) {   // even warps DFMA, odd warps DMMA
  const int warp = threadIdx.x >> 5;
  double s = 0;
  if (warp & 1) {
    double d[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) d[q] = 0.0;
    const double a = 1e-3 + seed * 1e-9 * threadIdx.x, b = 1e-3;
    for (int i = 0; i < ITERS; ++i) {
#pragma unroll
      for (int q = 0; q < 8; ++q) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d[2 * q]), "+d"(d[2 * q + 1]) : "d"(a), "d"(b));
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) s += d[q];
  } else {
    double x[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) x[q] = seed + 1e-9 * (threadIdx.x + q);
    const double y = 1.0000001 + seed * 1e-12;
    for (int i = 0; i < ITERS; ++i) {
#pragma unroll
      for (int q = 0; q < 8; ++q) x[q] = fma(x[q], y, 1e-9);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) s += x[q];
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <class F>
float best_ms(F launch) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int r = 0; r < 6; ++r) {
    cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (r > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return best;
}

int main() {
  int sm = 0, clk = 0; cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0); cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  const int threads = 256, blocks = sm * 8;
  double* out; cudaMalloc(&out, (size_t)blocks * threads * sizeof(double));
  const double nthreads = (double)blocks * threads, nwarps = nthreads / 32;
  const float t_fma = best_ms([&] { dfma_kernel<<<blocks, threads>>>(out, 1.0); });
  const float t_mma8 = best_ms([&] { dmma_kernel<8><<<blocks, threads>>>(out, 1.0); });
  const float t_mma21 = best_ms([&] { dmma_kernel<21><<<blocks, threads>>>(out, 1.0); });
  const float t_mix = best_ms([&] { mixed_kernel<<<blocks, threads>>>(out, 1.0); });
  const double fma_tf = nthreads * ITERS * 8 * 2 / (t_fma * 1e-3) / 1e12;
  const double mma8_tf = nwarps * ITERS * 8 * 512.0 / (t_mma8 * 1e-3) / 1e12;      // m8n8k4: 8*8*4*2 = 512 flop per warp instruction
  const double mma21_tf = nwarps * ITERS * 21 * 512.0 / (t_mma21 * 1e-3) / 1e12;
  const double mix_fma_tf = (nthreads / 2) * ITERS * 8 * 2 / (t_mix * 1e-3) / 1e12, mix_mma_tf = (nwarps / 2) * ITERS * 8 * 512.0 / (t_mix * 1e-3) / 1e12;
  printf("{\"sm_count\": %d, \"clock_khz\": %d, \"dfma_tflops\": %.3f, \"dmma_m8n8k4_tflops_8acc\": %.3f, \"dmma_m8n8k4_tflops_21acc\": %.3f, "
         "\"mixed_dfma_tflops\": %.3f, \"mixed_dmma_tflops\": %.3f, \"dmma_cycles_per_instr_per_subcore\": %.2f, \"err\": \"%s\"}\n",
         sm, clk, fma_tf, mma8_tf, mma21_tf, mix_fma_tf, mix_mma_tf,
         (t_mma21 * 1e-3) * (clk * 1e3) / ((nwarps / (sm * 4)) * ITERS * 21), cudaGetErrorString(cudaGetLastError()));
  return 0;
}
