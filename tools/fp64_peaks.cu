// Microbenchmark: measured FP64 throughput ceilings of one GPU -- the denominators of a second roofline of the residual / solver
// kernels next to the data-sheet figures bench.py divides by:
//   * DFMA (SIMT FP64 pipe): every thread runs 8 independent FMA chains;
//   * DMMA, per FP64 tensor shape (mma.sync m8n8k4, and the sm_90 shapes m16n8k4 / m16n8k8 / m16n8k16): every warp runs
//     8 / 21 independent accumulator fragments (21 = the vision tile's upper block triangle);
//   * both together (alternating warps), to see whether the two pipes overlap.  The DMMA warps of the mixed kernel do the
//     same FLOPs for every shape (fewer iterations for the wider ones), so its time compares the shapes' cost on the shared
//     pipe directly.
// Timed with CUDA events over a grid that fills all SMs (SM count x 8 CTAs x 256 threads), best of 5.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peaks fp64_peaks.cu && ./fp64_peaks > fp64_peaks.json
#include <cstdio>
#include <cuda_runtime.h>
#include "fp64_mma.cuh"

constexpr int ITERS = 4096;

// Iterations of the mixed kernel's DMMA warps: the FLOPs of ITERS m8n8k4 steps, whatever the shape.
template <Shape S> __host__ __device__ constexpr int mixed_iters() { return (int)(ITERS * Mma<M8N8K4>::FLOP / Mma<S>::FLOP); }

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

template <Shape S, int NACC>
__global__ void dmma_kernel(double* out, double seed) {
  constexpr int ACC = Mma<S>::ACC;
  double d[ACC * NACC];
#pragma unroll
  for (int q = 0; q < ACC * NACC; ++q) d[q] = 0.0;
  const double a = 1e-3 + seed * 1e-9 * threadIdx.x, b = 1e-3;
  for (int i = 0; i < ITERS; ++i) {
#pragma unroll
    for (int q = 0; q < NACC; ++q) Mma<S>::run(d + ACC * q, a, b);
  }
  double s = 0;
#pragma unroll
  for (int q = 0; q < ACC * NACC; ++q) s += d[q];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <Shape S>
__global__ void mixed_kernel(double* out, double seed) {   // even warps DFMA, odd warps DMMA
  constexpr int ACC = Mma<S>::ACC;
  const int warp = threadIdx.x >> 5;
  double s = 0;
  if (warp & 1) {
    double d[8 * ACC];
#pragma unroll
    for (int q = 0; q < 8 * ACC; ++q) d[q] = 0.0;
    const double a = 1e-3 + seed * 1e-9 * threadIdx.x, b = 1e-3;
    for (int i = 0; i < mixed_iters<S>(); ++i) {
#pragma unroll
      for (int q = 0; q < 8; ++q) Mma<S>::run(d + ACC * q, a, b);
    }
#pragma unroll
    for (int q = 0; q < 8 * ACC; ++q) s += d[q];
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

struct Ctx { int sm, clk, blocks, threads; double nthreads, nwarps; double* out; };

// Prints one shape's rows: alone with 8 and 21 accumulators, and mixed with DFMA warps.
template <Shape S>
void shape_rows(const Ctx& c, bool last) {
  const float t8 = best_ms([&] { dmma_kernel<S, 8><<<c.blocks, c.threads>>>(c.out, 1.0); });
  const float t21 = best_ms([&] { dmma_kernel<S, 21><<<c.blocks, c.threads>>>(c.out, 1.0); });
  const float tmix = best_ms([&] { mixed_kernel<S><<<c.blocks, c.threads>>>(c.out, 1.0); });
  const double f = Mma<S>::FLOP;
  const double tf8 = c.nwarps * ITERS * 8 * f / (t8 * 1e-3) / 1e12, tf21 = c.nwarps * ITERS * 21 * f / (t21 * 1e-3) / 1e12;
  const double mix_mma = (c.nwarps / 2) * mixed_iters<S>() * 8 * f / (tmix * 1e-3) / 1e12;
  const double mix_fma = (c.nthreads / 2) * ITERS * 8 * 2 / (tmix * 1e-3) / 1e12;
  printf("    \"%s\": {\"tflops_8acc\": %.3f, \"tflops_21acc\": %.3f, \"mixed_dmma_tflops\": %.3f, \"mixed_dfma_tflops\": %.3f, "
         "\"mixed_ms\": %.4f, \"cycles_per_instr_per_subcore_21acc\": %.2f}%s\n",
         Mma<S>::name, tf8, tf21, mix_mma, mix_fma, tmix,
         (t21 * 1e-3) * (c.clk * 1e3) / ((c.nwarps / (c.sm * 4)) * ITERS * 21), last ? "" : ",");
}

int main() {
  Ctx c{};
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  cudaDeviceGetAttribute(&c.sm, cudaDevAttrMultiProcessorCount, 0); cudaDeviceGetAttribute(&c.clk, cudaDevAttrClockRate, 0);
  c.threads = 256; c.blocks = c.sm * 8;
  cudaMalloc(&c.out, (size_t)c.blocks * c.threads * sizeof(double));
  c.nthreads = (double)c.blocks * c.threads; c.nwarps = c.nthreads / 32;
  const float t_fma = best_ms([&] { dfma_kernel<<<c.blocks, c.threads>>>(c.out, 1.0); });
  printf("{\"device\": \"%s\", \"sm_count\": %d, \"clock_khz\": %d, \"dfma_tflops\": %.3f,\n  \"dmma\": {\n", prop.name, c.sm, c.clk,
         c.nthreads * ITERS * 8 * 2 / (t_fma * 1e-3) / 1e12);
  shape_rows<M8N8K4>(c, false);
  shape_rows<M16N8K4>(c, false);
  shape_rows<M16N8K8>(c, false);
  shape_rows<M16N8K16>(c, true);
  printf("  },\n  \"err\": \"%s\"}\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
