// Lane-private parking of FP64 register arrays in the warp's shared-memory park (sm_90a: 227 KB of shared memory per block).
// Double j of lane l lives at park[j * 32 + l]: a warp's 64-bit access touches 256 consecutive bytes, so every park / unpark
// is conflict-free.  A lane only ever reads back what it wrote itself, so no fence or warp barrier is needed between the two.
#pragma once

namespace icc {

// p = warp park + lane + 32 * (first double)
template <int N>
__device__ __forceinline__ void park_st(double* __restrict__ p, const double (&v)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) p[32 * i] = v[i];
}
template <int N>
__device__ __forceinline__ void park_ld(const double* __restrict__ p, double (&v)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = p[32 * i];
}

}  // namespace icc
