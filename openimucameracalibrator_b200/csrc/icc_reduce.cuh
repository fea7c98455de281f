// Warp and block reductions of the upstream kernels, and the packed normal equations the in-kernel minimisers reduce with them.
// Device only (warp shuffles): the per-thread arithmetic that the CPU tests compile lives in icc_small_linalg.cuh.
// Every reduction here has one fixed order of additions, so a kernel that uses nothing else is bit-repeatable run to run.
#pragma once
#include "icc_device_math.cuh"

namespace icc {

// xor butterfly over the warp: every lane returns the result
ICC_D double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
ICC_D double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// tot[k] = sum over the block of every thread's s[k]: warp_sum per warp, then thread k adds the warps in warp order.  Called by the
// whole block (a multiple of 32 threads, at least K); red holds one row per warp; tot is valid in every thread on return.
template <int K>
ICC_D void block_sums(const double (&s)[K], double (*red)[K], double* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double v = warp_sum(s[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) { double v = 0.0; for (int w = 0; w < nw; ++w) v += red[w][threadIdx.x]; tot[threadIdx.x] = v; }
  __syncthreads();
}

// Normal equations of a least-squares problem with N unknowns as one vector of sums: the upper triangle of J^T J row by row, then
// J^T r, then r^T r.
constexpr int normal_equation_sums(int n) { return n * (n + 1) / 2 + n + 1; }

template <int N>
ICC_D void normal_equation_row(double (&s)[normal_equation_sums(N)], const double (&J)[N], double r) {   // adds one residual row
  int c = 0;
#pragma unroll
  for (int p = 0; p < N; ++p)
#pragma unroll
    for (int q = p; q < N; ++q) s[c++] += J[p] * J[q];
#pragma unroll
  for (int p = 0; p < N; ++p) s[c + p] += J[p] * r;
  s[c + N] += r * r;
}

// the reduced sums as H = J^T J (symmetric), g = J^T r and cost = r^T r / 2 of a minimiser with LD >= N unknowns; rows and columns
// from N on are zero
template <int N, int LD>
ICC_D void unpack_normal_equations(const double* tot, double (&H)[LD][LD], double (&g)[LD], double& cost) {
  constexpr int T = N * (N + 1) / 2;
  for (int p = 0; p < LD; ++p) { g[p] = p < N ? tot[T + p] : 0.0; for (int q = 0; q < LD; ++q) H[p][q] = 0.0; }
  int c = 0;
  for (int p = 0; p < N; ++p) for (int q = p; q < N; ++q) { H[p][q] = tot[c]; H[q][p] = tot[c]; ++c; }
  cost = 0.5 * tot[T + N];
}

}  // namespace icc
