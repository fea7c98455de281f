// Device helpers shared by the persistent residual kernels (icc_vision_tmem.cu, icc_imu_tmem.cu): the FP64 tensor-core symmetric
// rank-k update of a column-major shared-memory tile, and the scatter of the finished fragments into the packed banded + bordered
// normal equations.
#pragma once
#include "icc_device_math.cuh"
#include <stdint.h>

namespace icc {

constexpr int TILE_LD = 36;            // rows per tile column (32 + 4 pad: conflict-free fragment loads)
constexpr int TILE_COLS = 48;

// one 8 x 8 block: c (m8n8 fragment) += a b^T over one k-step of 4 rows
__device__ __forceinline__ void tile_mma_f64(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// two 8 x 8 blocks of one block column in one m16n8k4: A rows g and g + 8 are a0 and a1, so (c0, c1) += a0 b^T and (c2, c3) += a1 b^T
// are the m8n8 fragments of the two blocks in the same lane layout as tile_mma_f64's.  One DMMA.16x8x4 holds the H100's FP64 pipe
// as long as one DMMA.8x8x4 (16 cycles per SM sub-partition, tools/fp64_peaks.cu; DESIGN §5), so a pair costs half.
__device__ __forceinline__ void tile_mma2_f64(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3) : "d"(a0), "d"(a1), "d"(b));
}

// acc += T^T T over tile rows [4 k0, 4 k1), NB column blocks of 8: the upper block triangle, NB (NB + 1) / 2 fragments of 2 doubles
// stored block column by block column (bj outer, bi = 0..bj inner).  Within a block column the blocks bi = 2p and 2p + 1 are
// adjacent fragments and share one m16n8k4; the diagonal block of an even block column is left over and takes one m8n8k4
// (NB = 6: 9 + 3 instructions per k-step instead of 21).
template <int NB>
__device__ __forceinline__ void tile_syrk(const double* __restrict__ tile, int k0, int k1, double (&acc)[NB * (NB + 1)]) {
  const int lane = threadIdx.x & 31;
  const double* base = tile + (lane >> 2) * TILE_LD + (lane & 3);
  for (int s = k0; s < k1; ++s) {
    double f[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) f[b] = base[(8 * b) * TILE_LD + 4 * s];
    int idx = 0;
#pragma unroll
    for (int bj = 0; bj < NB; ++bj) {
#pragma unroll
      for (int bi = 0; bi < bj; bi += 2) { tile_mma2_f64(acc[2 * idx], acc[2 * idx + 1], acc[2 * idx + 2], acc[2 * idx + 3], f[bi], f[bi + 1], f[bj]); idx += 2; }
      if (bj % 2 == 0) { tile_mma_f64(acc[2 * idx], acc[2 * idx + 1], f[bj], f[bj]); ++idx; }
    }
  }
}

struct NeLayout { double* ne; int64_t off_E, off_C, off_g, off_cost; int nk, nb, ldb; };

// Scatter one finished tile from the register fragments: one RED.ADD.F64 per entry of the upper triangle.  Kept branch-free
// (selected addresses, predicated RED) and specialised per block at compile time: block columns < GEN0 hold spline-knot columns
// only, which always land in the band; the residual column (gradient / cost, gidx == -2) only exists in the LAST block column.
// gidx: tile column -> solver column, -1 = constant / padding, -2 = residual column.
template <int NB, int GEN0>
__device__ __forceinline__ void tile_flush(const NeLayout& L, const int* __restrict__ gidx, const double (&acc)[NB * (NB + 1)]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t2 = 2 * (lane & 3);
  int gI[NB], gJ[NB][2];
#pragma unroll
  for (int b = 0; b < NB; ++b) { gI[b] = gidx[8 * b + g]; const int2 j2 = *reinterpret_cast<const int2*>(gidx + 8 * b + t2); gJ[b][0] = j2.x; gJ[b][1] = j2.y; }
  const int ldbm1 = L.ldb - 1;
  int idx = 0;
#pragma unroll
  for (int bj = 0; bj < NB; ++bj)                                                 // tile_syrk's fragment order
#pragma unroll
    for (int bi = 0; bi <= bj; ++bi) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        double v = acc[2 * idx + e];
        const int gi = gI[bi], gj = gJ[bj][e];
        bool ok = gi != -1 && gj != -1 && (bi < bj || g <= t2 + e);
        const int lo = min(gi, gj), hi = max(gi, gj);
        int64_t off = (int64_t)lo * ldbm1 + hi;                                  // band: lo * ldb + (hi - lo)
        if (bj >= GEN0) {                                                         // these tile columns may be border columns
          if (hi >= L.nk) off = lo < L.nk ? L.off_E + (int64_t)lo * L.nb + (hi - L.nk) : L.off_C + (int64_t)(hi - L.nk) * L.nb + (lo - L.nk);
        }
        if (bj == NB - 1) {                                                       // the residual column lives in the last block column
          if (gj == -2) { off = gi == -2 ? L.off_cost : L.off_g + gi; if (gi == -2) v *= 0.5; }   // r^T r = 2 cost ; J^T r
          else if (gi == -2) ok = false;
        }
        if (ok) atomicAdd(L.ne + off, v);
      }
      ++idx;
    }
}

}  // namespace icc
