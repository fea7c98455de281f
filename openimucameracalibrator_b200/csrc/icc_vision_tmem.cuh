// Rolling-shutter reprojection residuals + analytic Jacobians + J^T J / J^T r reduction: the vision items of the persistent, shared-memory-parking evaluation kernel (icc_eval_tmem.cu, sm_90a).
//
// Same arithmetic contract as vision_kernel<1> of icc_eval.cu (reference: RSReprojectionCostFunctorSplit<6>::operator(),
// basalt_spline/ceres_calib_split_residuals.h:319-402, under Ceres autodiff + LieLocalParameterization), re-mapped to the machine:
//
//  * ONE persistent CTA of eight warps per SM (two per SM sub-partition).  The 21 FP64 tensor-core accumulator fragments (42 doubles
//    per lane) stay in registers for the warp's whole run, next to the per-corner spline chain.
//  * Both rows of a corner are evaluated in ONE pass (icc_vision_rows.cuh): the x row goes to the warp's shared-memory tile, the
//    y row (36 doubles, R^3 block factored) goes entry by entry to the warp's lane-private shared-memory park (icc_park.cuh) and is
//    expanded into the same tile after the x rows have been contracted.  Neither row is held in registers, so chain and
//    accumulators fit in 255 registers together and nothing spills; the park is 36 instead of 78 doubles per lane, which is what
//    lets eight warps' tiles and parks fit in one block's shared memory.
//  * The corners of all frames form ONE packed stream (frames padded to a multiple of 4 = one tensor-core k-step) that is cut into
//    equal runs of 32-lane chunks, one run per warp: no partial last wave, no half-empty chunk at the end of a 144-corner frame.
//    A chunk may straddle two frames (two staged knot windows, lanes pick theirs); the k-steps of the first frame finish its
//    tile, which is flushed, before the k-steps of the second start a new one.
//  * flush: one RED.ADD.F64 per tile entry into the packed banded+bordered normal equations (L2-resident), with the row/column
//    index maps preloaded per lane.
#pragma once
#include "icc_kernels.h"
#include "icc_tile_common.cuh"
#include "icc_park.cuh"
#include "icc_vision_rows.cuh"

namespace icc {
namespace tmv {

constexpr int VW = 8;                  // warps per CTA: two per SM sub-partition
constexpr int LDT = TILE_LD, TCOLS = TILE_COLS;   // 44 tile columns used
constexpr int PARK_N = YR_N;           // park doubles per lane: the y row
constexpr int NBLK = 21;               // upper block triangle of 6 x 6 blocks of 8 columns

struct WarpSlot {
  FrameWin win[2];
  int gidx[2][TCOLS];                  // tile column -> solver column; -1 = constant / padding, -2 = residual column
  int finfo[2][4];                     // per staged frame: padded stream offset, first corner, corner count
};

// incr / n_incr: the evaluated state's SO(3) increment table (incr_table_entry) and its entry count
struct StageArgs { const double* incr; const double4* so3; const double4* r3; const int* so3_col; const int* r3_col; int n_incr, col_tic, col_ld; };

// Stage the knot windows of one frame: all lanes copy the five SO(3) increments (log, unit axis, Jr^-1) from the increment table,
// lane 0 takes the first knot, lanes 8..13 the R^3 knots, all lanes the tile-column -> solver-column map.  Every load is issued before
// the first store, so a window costs one L2 round trip and no arithmetic on the lanes.
__device__ __noinline__ void stage_frame(WarpSlot* slot, int w, VisFrame F, StageArgs A) {
  const int lane = threadIdx.x & 31;
  double inc[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { const int e = lane + 32 * k; inc[k] = e < WIN_INCR_DOUBLES ? A.incr[incr_table_index(e, F.s_so3, A.n_incr)] : 0.0; }
  double4 k4 = make_double4(0, 0, 0, 1);
  if (lane == 0) k4 = A.so3[F.s_so3];
  else if (lane >= 8 && lane < 14) k4 = A.r3[F.s_r3 + lane - 8];
  int g[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int c = lane + 32 * j;
    g[j] = -1;
    if (c < 18) { const int b = A.so3_col[F.s_so3 + c / 3]; g[j] = b < 0 ? -1 : b + c % 3; }
    else if (c < 36) { const int b = A.r3_col[F.s_r3 + (c - 18) / 3]; g[j] = b < 0 ? -1 : b + (c - 18) % 3; }
    else if (c < 42) g[j] = A.col_tic < 0 ? -1 : A.col_tic + (c - 36);
    else if (c == 42) g[j] = A.col_ld;
    else if (c == VIS_RES_COL) g[j] = -2;
  }
  __syncwarp();                                   // every lane is done with whatever this window slot held before
  FrameWin& W = slot->win[w];
  double* wi = win_incr(W);
#pragma unroll
  for (int k = 0; k < 3; ++k) if (lane + 32 * k < WIN_INCR_DOUBLES) wi[lane + 32 * k] = inc[k];
  if (lane == 0) { W.q0 = q4(k4.x, k4.y, k4.z, k4.w); W.u_so3 = F.u_so3; W.u_r3 = F.u_r3; slot->finfo[w][0] = F.poff; slot->finfo[w][1] = F.c0; slot->finfo[w][2] = F.cn; }
  if (lane >= 8 && lane < 14) W.p[lane - 8] = v3(k4.x, k4.y, k4.z);
#pragma unroll
  for (int j = 0; j < 2; ++j) if (lane + 32 * j < TCOLS) slot->gidx[w][lane + 32 * j] = g[j];
  __syncwarp();
}

// One tile part: rows [4 k0, 4 k1) of the chunk belong to one frame.  acc holds the frame's accumulators (zero when its tile starts
// here); last: the frame's tile (or the item) ends here: scatter them and zero them for the next frame.
ICC_D void tile_part(const NeLayout& L, double* __restrict__ tile, int k0, int k1, bool last, const int* __restrict__ gidx, double (&acc)[2 * NBLK], double* ta, int lane) {
  tile_syrk<6>(tile, k0, k1, acc);                       // x rows
  __syncwarp();
  {                                               // expand the parked y rows of this part into the tile (same rows)
    const bool mine = lane >= 4 * k0 && lane < 4 * k1;
    double* yrow = tile + lane;
    double h[18];
    park_ld(ta, h);
    if (mine) {
#pragma unroll
      for (int c = 0; c < 18; ++c) yrow[c * LDT] = h[c];
    }
    park_ld(ta + 32 * 18, h);                   // [m_t 0..2 | Dp 3..5 | om 6..8 | ld 9 | r 10 | cc 11..16 | pad]
    if (mine) {
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        yrow[(18 + 3 * j + 0) * LDT] = -h[11 + j] * h[0]; yrow[(18 + 3 * j + 1) * LDT] = -h[11 + j] * h[1]; yrow[(18 + 3 * j + 2) * LDT] = -h[11 + j] * h[2];
      }
      yrow[36 * LDT] = -h[3]; yrow[37 * LDT] = -h[4]; yrow[38 * LDT] = -h[5];
      yrow[39 * LDT] = h[6]; yrow[40 * LDT] = h[7]; yrow[41 * LDT] = h[8];
      yrow[42 * LDT] = h[9];
      yrow[VIS_RES_COL * LDT] = h[10];
    }
  }
  __syncwarp();
  tile_syrk<6>(tile, k0, k1, acc);                       // y rows
  __syncwarp();
  if (last) {
    tile_flush<6, 4>(L, gidx, acc);
#pragma unroll
    for (int i = 0; i < 2 * NBLK; ++i) acc[i] = 0.0;
  }
}

// shared-memory constants of the vision items (written once per CTA)
ICC_D void init_const(VisConst* K, const DeviceProblem& P, const DeviceState& S, int model) {
  if (threadIdx.x < MAX_INTR) K->intr[threadIdx.x] = S.glob[G_CAM_INTR + threadIdx.x];
  if (threadIdx.x == 32) {
    const Q4 q_ic = q4(S.glob[G_TIC + 0], S.glob[G_TIC + 1], S.glob[G_TIC + 2], S.glob[G_TIC + 3]);
    K->Ric = qmat(q_ic); K->tic = v3(S.glob[G_TIC + 4], S.glob[G_TIC + 5], S.glob[G_TIC + 6]);
    K->ld = S.glob[G_LD]; K->model = model; K->fov = P.dispatch_fov;
  }
}

// One item = one contiguous run of 32-lane chunks of the packed corner stream, processed by one warp.
template <int MODEL>
ICC_D void run_item(const DeviceProblem& P, const TangentMeas& T, const DeviceState& S, const VisConst* K, WarpSlot* slot, double* __restrict__ tile, double* ta, const NeLayout& L, const VisItem it, double* __restrict__ res_out, int lane, int rounds, int bar_id, int bar_n) {
  StageArgs A; A.incr = P.incr; A.n_incr = P.n_so3 - 1; A.so3 = S.so3; A.r3 = S.r3; A.so3_col = P.so3_col; A.r3_col = P.r3_col; A.col_tic = P.col_tic; A.col_ld = P.col_ld;
  double acc[2 * NBLK];                           // the current frame's tile accumulators, in registers for the whole run
#pragma unroll
  for (int i = 0; i < 2 * NBLK; ++i) acc[i] = 0.0;
  {
    int f = it.vf0, pos = it.pos_begin, cur = 0;
    stage_frame(slot, cur, P.vframes[f], A);
    int endF = min(P.vframes[f + 1].poff, it.pos_end);
    while (pos < it.pos_end) {
      if (rounds > 0) { asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); --rounds; }   // loose lockstep of the warps of a group: instruction-cache locality (icc_eval_tmem.cu)
      if (pos == endF) {                          // the previous chunk finished its frame exactly at the chunk boundary
        ++f;
        stage_frame(slot, cur, P.vframes[f], A);
        endF = min(P.vframes[f + 1].poff, it.pos_end);
      }
      const int nA = min(32, endF - pos);
      int nB = 0, endB = 0;
      if (nA < 32 && endF < it.pos_end) {         // the frame ends inside this chunk: the remaining lanes start the next frame
        endB = min(P.vframes[f + 2].poff, it.pos_end);
        nB = min(32 - nA, endB - endF);
        stage_frame(slot, cur ^ 1, P.vframes[f + 1], A);
      }
      const int n = nA + nB;
      // ---- SIMT pass: both rows of this lane's corner --------------------------------------------------------------
      {
        const bool inA = lane < nA;
        const int w = inA ? cur : cur ^ 1;
        const int rel = inA ? pos + lane - slot->finfo[w][0] : lane - nA;
        double* xrow = tile + lane;
        if (lane < n && rel < slot->finfo[w][2]) {
          const int c = slot->finfo[w][1] + rel;
          const double2 ob = P.uv[c];
          const double4 X = P.board[P.pid[c]];
          double r0, r1;
          if constexpr (MODEL == VIS_TANGENT) vision_corner_rows<MODEL>(slot->win[w], *K, v3(X.x, X.y, X.z), ob.x, ob.y, T.bear[c], T.ok[c] != 0, T.s, xrow, LDT, ta, 32, r0, r1);
          else vision_corner_rows<MODEL>(slot->win[w], *K, v3(X.x, X.y, X.z), ob.x, ob.y, xrow, LDT, ta, 32, r0, r1);   // y row straight to the park
          if (res_out) { res_out[2 * c] = r0; res_out[2 * c + 1] = r1; }
        } else {                                  // padding lane of a frame whose corner count is not a multiple of 4, or beyond the chunk
#pragma unroll
          for (int c = 0; c <= VIS_RES_COL; ++c) xrow[c * LDT] = 0.0;
#pragma unroll
          for (int c = 0; c < PARK_N; ++c) ta[32 * c] = 0.0;
        }
      }
      __syncwarp();
      // ---- tensor-core passes: the rows of the frame that ends first, then (straddling chunk) the rows of the next frame --------
      // (a straddling chunk always ends the first frame in part 0, so part 1 starts from zeroed accumulators)
#pragma unroll 1
      for (int part = 0; part < (nB ? 2 : 1); ++part) {
        const int k0 = part ? nA >> 2 : 0, k1 = part ? n >> 2 : nA >> 2;
        const bool last = part ? endF + nB == endB : pos + nA == endF;
        tile_part(L, tile, k0, k1, last, slot->gidx[part ? cur ^ 1 : cur], acc, ta, lane);
      }
      if (nB) { ++f; cur ^= 1; endF = endB; }
      pos += n;
    }
  }
  while (rounds-- > 0) asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory");
}

}  // namespace tmv
}  // namespace icc
