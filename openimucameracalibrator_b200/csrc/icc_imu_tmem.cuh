// Accelerometer + gyroscope residuals, analytic Jacobians and J^T J / J^T r reduction: the IMU items of the persistent, shared-memory-parking evaluation kernel (icc_eval_tmem.cu, sm_90a).
//
// Same arithmetic contract as imu_kernel<true, 0> of icc_eval.cu (reference: AccelerationCostFunctorSplit<6> / GyroCostFunctorSplit<6>,
// basalt_spline/ceres_calib_split_residuals.h:52-93,133-169, under Ceres autodiff + LieLocalParameterization) for the column set of
// the hot CLI's stage 1 with fixed biases; the wider column sets (bias knots, IMU intrinsics, time offset) stay on imu_kernel.
// Machine mapping = icc_vision_tmem.cu:
//  * ONE persistent CTA of eight warps per SM (two per SM sub-partition).  The 15 + 6 FP64 tensor-core accumulator fragments of
//    the two tiles (accelerometer 40 columns, gyroscope 24; 42 doubles per lane) stay in registers for the warp's whole run, next
//    to the per-sample spline chain;
//  * the three rows of a sensor are evaluated in ONE pass (icc_imu_rows.cuh): row 0 goes to the warp's shared-memory tile, rows 1
//    and 2 go entry by entry to the warp's lane-private shared-memory park (icc_park.cuh; 43 / 38 doubles) and are expanded into
//    the same tile after the previous row has been contracted.  The park holds only these deferred rows, which is what lets
//    eight warps' tiles and parks fit in one block's shared memory;
//  * the samples of all knot-interval cells form ONE packed stream (cells padded to a multiple of 4 = one tensor-core k-step) cut into
//    equal runs of 32-lane chunks, one run per warp: a 50-sample cell (1 kHz, dt = 0.05 s) no longer costs two passes with 18 of 32
//    lanes idle in the second; a chunk may straddle two cells (two staged windows, lanes pick theirs).
#pragma once
#include "icc_imu_rows.cuh"
#include "icc_kernels.h"
#include "icc_tile_common.cuh"
#include "icc_park.cuh"

namespace icc {
namespace tmi {

constexpr int IW = 8;                        // warps per CTA: two per SM sub-partition
constexpr int LDT = TILE_LD, TCOLS = TILE_COLS;
constexpr int PARK_N = ACC_PARK;             // park doubles per lane: the deferred rows 1 and 2 of one sensor
static_assert(ACC_PARK <= PARK_N && GYR_PARK <= PARK_N, "park layout");

struct ImuSlot {
  ImuWin win[2];
  int gidxA[2][TCOLS];                       // accelerometer tile column -> solver column; -1 constant / padding, -2 residual
  int gidxG[2][24];
  int cinfo[2][8];                           // per staged cell: padded stream offset, first sample, sample count, s_so3, s_r3, s_ba, s_bg
};
// incr / n_incr: the evaluated state's SO(3) increment table (incr_table_entry) and its entry count
struct ImuStageArgs { const double* incr; const double4* so3; const double4* r3; const double4* ba; const double4* bg; const int* so3_col; const int* r3_col; int n_incr, col_g; };

// Stage the knot windows of one cell: all lanes copy the five SO(3) increments from the increment table, lane 0 takes the first knot,
// lanes 8..13 the R^3 knots, lanes 16..18 / 20..22 the bias knots, all lanes the column maps.  Every load is issued before the first
// store (one L2 round trip, no arithmetic).
// slot_sa: the slot's shared-window address.  A generic slot pointer would keep one more register live across the run loop's calls,
// whose callee-saved range leaves the run loop none to spare next to its register accumulators.
__device__ __noinline__ void stage_cell(unsigned slot_sa, int w, ImuCellP C, ImuStageArgs A) {
  ImuSlot* slot = static_cast<ImuSlot*>(__cvta_shared_to_generic(slot_sa));
  const int lane = threadIdx.x & 31;
  double inc[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { const int e = lane + 32 * k; inc[k] = e < WIN_INCR_DOUBLES ? A.incr[incr_table_index(e, C.s_so3, A.n_incr)] : 0.0; }
  double4 k4 = make_double4(0, 0, 0, 1);
  if (lane == 0) k4 = A.so3[C.s_so3];
  else if (lane >= 8 && lane < 14) k4 = A.r3[C.s_r3 + lane - 8];
  else if (lane >= 16 && lane < 19) k4 = A.ba[C.s_ba + lane - 16];
  else if (lane >= 20 && lane < 23) k4 = A.bg[C.s_bg + lane - 20];
  int g[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int c = lane + 32 * j;
    g[j] = -1;
    if (c < 18) { const int b = A.so3_col[C.s_so3 + c / 3]; g[j] = b < 0 ? -1 : b + c % 3; }
    else if (c < 36) { const int b = A.r3_col[C.s_r3 + (c - 18) / 3]; g[j] = b < 0 ? -1 : b + (c - 18) % 3; }
    else if (c < 39) g[j] = A.col_g < 0 ? -1 : A.col_g + (c - 36);
    else if (c == ACC_RES_COL) g[j] = -2;
  }
  __syncwarp();
  ImuWin& W = slot->win[w];
  double* wi = win_incr(W.f);
#pragma unroll
  for (int k = 0; k < 3; ++k) if (lane + 32 * k < WIN_INCR_DOUBLES) wi[lane + 32 * k] = inc[k];
  if (lane == 0) {
    W.f.q0 = q4(k4.x, k4.y, k4.z, k4.w); W.f.u_so3 = 0.0; W.f.u_r3 = 0.0;
    slot->cinfo[w][0] = C.poff; slot->cinfo[w][1] = C.i0; slot->cinfo[w][2] = C.n; slot->cinfo[w][3] = C.s_so3; slot->cinfo[w][4] = C.s_r3; slot->cinfo[w][5] = C.s_ba; slot->cinfo[w][6] = C.s_bg;
  }
  if (lane >= 8 && lane < 14) W.f.p[lane - 8] = v3(k4.x, k4.y, k4.z);
  if (lane >= 16 && lane < 19) W.ba[lane - 16] = v3(k4.x, k4.y, k4.z);
  if (lane >= 20 && lane < 23) W.bg[lane - 20] = v3(k4.x, k4.y, k4.z);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int c = lane + 32 * j;
    if (c < TCOLS) slot->gidxA[w][c] = g[j];
    if (c < 24) slot->gidxG[w][c] = c < 18 ? g[j] : (c == GYR_RES_COL ? -2 : -1);
  }
  __syncwarp();
}

// accelerometer tile part (rows [4 k0, 4 k1) of the chunk belong to one cell): rows 0, 1, 2 contracted one after the other.  acc
// holds the cell's accumulators (zero when its tile starts here); last: the cell's tile (or the item) ends here: scatter them and
// zero them for the next cell.
ICC_D void accel_part(const NeLayout& L, const ImuConst& K, double* __restrict__ tile, int k0, int k1, bool last, const int* __restrict__ gidx, double (&acc)[30], double* ta, int lane) {
  tile_syrk<5>(tile, k0, k1, acc);
  const bool mine = lane >= 4 * k0 && lane < 4 * k1;
#pragma unroll 1
  for (int k = 1; k <= 2; ++k) {
    __syncwarp();
    {
      double so3[18], tail[7];                                   // tail = [q (4) | r1 | r2 | u_r3]
      park_ld(ta + 32 * (k == 1 ? 0 : 18), so3);
      park_ld(ta + 32 * 36, tail);
      if (mine) imu_accel_row_expand(so3, q4(tail[0], tail[1], tail[2], tail[3]), k == 1 ? tail[4] : tail[5], tail[6], K, k, tile + lane, LDT);
    }
    __syncwarp();
    tile_syrk<5>(tile, k0, k1, acc);
  }
  __syncwarp();
  if (last) {
    tile_flush<5, 4>(L, gidx, acc);
#pragma unroll
    for (int i = 0; i < 30; ++i) acc[i] = 0.0;
  }
}

ICC_D void gyro_part(const NeLayout& L, double* __restrict__ tile, int k0, int k1, bool last, const int* __restrict__ gidx, double (&acc)[12], double* ta, int lane) {
  tile_syrk<3>(tile, k0, k1, acc);
  const bool mine = lane >= 4 * k0 && lane < 4 * k1;
#pragma unroll 1
  for (int k = 1; k <= 2; ++k) {
    __syncwarp();
    {
      double so3[18], tail[2];
      park_ld(ta + 32 * (k == 1 ? 0 : 18), so3);
      park_ld(ta + 32 * 36, tail);
      if (mine) {
        double* row = tile + lane;
#pragma unroll
        for (int c = 0; c < 18; ++c) row[c * LDT] = so3[c];
        row[GYR_RES_COL * LDT] = k == 1 ? tail[0] : tail[1];
#pragma unroll
        for (int c = GYR_RES_COL + 1; c < 24; ++c) row[c * LDT] = 0.0;
      }
    }
    __syncwarp();
    tile_syrk<3>(tile, k0, k1, acc);
  }
  __syncwarp();
  if (last) {
    tile_flush<3, 2>(L, gidx, acc);
#pragma unroll
    for (int i = 0; i < 12; ++i) acc[i] = 0.0;
  }
}

ICC_D void init_const(ImuConst* K, const DeviceProblem& P, const DeviceState& S) {
  if (threadIdx.x == 64) {
    const double* ai = S.glob + G_ACC_INTR; const double* gi = S.glob + G_GYR_INTR;
    // misalignment * scale matrices (utils/types.h:226-246)
    const double Ma[9] = {ai[3], -ai[0] * ai[4], ai[1] * ai[5], 0.0, ai[4], -ai[2] * ai[5], 0.0, 0.0, ai[5]};
    const double Mg[9] = {gi[6], -gi[0] * gi[7], gi[1] * gi[8], gi[3] * gi[6], gi[7], -gi[2] * gi[8], -gi[4] * gi[6], gi[5] * gi[7], gi[8]};
    for (int i = 0; i < 9; ++i) { K->Ma[i] = Ma[i]; K->Mg[i] = Mg[i]; }
    K->grav = v3(S.glob[G_GRAV], S.glob[G_GRAV + 1], S.glob[G_GRAV + 2]);
    K->w_acc = P.w_acc; K->w_gyr = P.w_gyr; K->idt2 = P.inv_r3_dt * P.inv_r3_dt; K->inv_so3_dt = P.inv_so3_dt;
    const double dto = S.glob[G_TOFF];        // time-offset increment [s] (0 unless the extension has been optimised)
    K->du_so3 = dto * P.inv_so3_dt; K->du_r3 = dto * P.inv_r3_dt; K->du_ba = dto * (1e9 / double(P.dt_ba_ns)); K->du_bg = dto * (1e9 / double(P.dt_bg_ns));
  }
}

// One item = one contiguous run of 32-lane chunks of the packed IMU sample stream, processed by one warp.  The warps of a lockstep
// group meet twice per chunk (before the accelerometer and before the gyroscope pass) at the group's one named barrier `bar_id`.
ICC_D void run_item(const DeviceProblem& P, const DeviceState& S, const ImuConst* K, ImuSlot* slot, double* __restrict__ tile, double* ta, const NeLayout& L, const VisItem it, double* __restrict__ res_out, int lane, int rounds, int bar_id, int bar_n) {
  const bool lock = rounds > 0;
  const unsigned slot_sa = (unsigned)__cvta_generic_to_shared(slot);
  ImuStageArgs A; A.incr = P.incr; A.n_incr = P.n_so3 - 1; A.so3 = S.so3; A.r3 = S.r3; A.ba = S.ba; A.bg = S.bg; A.so3_col = P.so3_col; A.r3_col = P.r3_col; A.col_g = P.col_g;
  double accA[30], accG[12];                  // the current cell's tile accumulators, in registers for the whole run
#pragma unroll
  for (int k = 0; k < 30; ++k) accA[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 12; ++k) accG[k] = 0.0;
  {
    int c = it.vf0, pos = it.pos_begin, cur = 0;
    stage_cell(slot_sa, cur, P.icells[c], A);
    int endC = min(P.icells[c + 1].poff, it.pos_end);
    while (pos < it.pos_end) {
      if (rounds > 0) { asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); --rounds; }   // loose lockstep of the warps of a group (instruction-cache locality)
      if (pos == endC) {
        ++c;
        stage_cell(slot_sa, cur, P.icells[c], A);
        endC = min(P.icells[c + 1].poff, it.pos_end);
      }
      const int nA = min(32, endC - pos);
      int nB = 0, endB = 0;
      if (nA < 32 && endC < it.pos_end) {
        endB = min(P.icells[c + 2].poff, it.pos_end);
        nB = min(32 - nA, endB - endC);
        stage_cell(slot_sa, cur ^ 1, P.icells[c + 1], A);
      }
      const int n = nA + nB;
      const bool inA = lane < nA;
      const int w = inA ? cur : cur ^ 1;
      const int rel = inA ? pos + lane - slot->cinfo[w][0] : lane - nA;
      const bool act = lane < n && rel < slot->cinfo[w][2];
      const int i = slot->cinfo[w][1] + rel;
      const bool lastA = pos + nA == endC, lastB = nB ? endC + nB == endB : false;
      // ---- accelerometer: SIMT pass, then three tensor-core passes per cell part ----------------------------------------
      {
        double* row0 = tile + lane;
        if (act) {
          const int64_t st = P.imu_t_ns[i];
          // CalcTimes (impl.h:763-788): u = (st % dt) / dt with the segment index known from the cell
          const double u_so3 = double(st - (int64_t)slot->cinfo[w][3] * P.dt_so3_ns) / double(P.dt_so3_ns) + K->du_so3;
          const double u_r3 = double(st - (int64_t)slot->cinfo[w][4] * P.dt_r3_ns) / double(P.dt_r3_ns) + K->du_r3;
          const double u_ba = double(st - (int64_t)slot->cinfo[w][5] * P.dt_ba_ns) / double(P.dt_ba_ns) + K->du_ba;
          double ra[3];
          imu_accel_rows(slot->win[w], *K, u_so3, u_r3, u_ba, v3(P.imu_acc[3 * i], P.imu_acc[3 * i + 1], P.imu_acc[3 * i + 2]), row0, LDT, ta, 32, ra);   // rows 1, 2 straight to the park
          if (res_out) { res_out[P.n_res_vis + 3 * i] = ra[0]; res_out[P.n_res_vis + 3 * i + 1] = ra[1]; res_out[P.n_res_vis + 3 * i + 2] = ra[2]; }
        } else {
#pragma unroll
          for (int cc = 0; cc <= ACC_RES_COL; ++cc) row0[cc * LDT] = 0.0;
#pragma unroll
          for (int cc = 0; cc < ACC_PARK; ++cc) ta[32 * cc] = 0.0;
        }
      }
      __syncwarp();
#pragma unroll 1
      for (int part = 0; part < (nB ? 2 : 1); ++part)
        accel_part(L, *K, tile, part ? nA >> 2 : 0, part ? n >> 2 : nA >> 2, part ? lastB : lastA, slot->gidxA[part ? cur ^ 1 : cur], accA, ta, lane);
      __syncwarp();
      // ---- gyroscope ------------------------------------------------------------------------------------------------------
      if (lock) asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory");
      {
        double* row0 = tile + lane;
        if (act) {
          const int64_t st = P.imu_t_ns[i];
          const double u_so3 = double(st - (int64_t)slot->cinfo[w][3] * P.dt_so3_ns) / double(P.dt_so3_ns) + K->du_so3;
          const double u_bg = double(st - (int64_t)slot->cinfo[w][6] * P.dt_bg_ns) / double(P.dt_bg_ns) + K->du_bg;
          double rg[3];
          imu_gyro_rows(slot->win[w], *K, u_so3, u_bg, v3(P.imu_gyr[3 * i], P.imu_gyr[3 * i + 1], P.imu_gyr[3 * i + 2]), row0, LDT, ta, 32, rg);
          if (res_out) { res_out[P.n_res_vis + P.n_res_acc + 3 * i] = rg[0]; res_out[P.n_res_vis + P.n_res_acc + 3 * i + 1] = rg[1]; res_out[P.n_res_vis + P.n_res_acc + 3 * i + 2] = rg[2]; }
        } else {
#pragma unroll
          for (int cc = 0; cc < 24; ++cc) row0[cc * LDT] = 0.0;
#pragma unroll
          for (int cc = 0; cc < GYR_PARK; ++cc) ta[32 * cc] = 0.0;
        }
      }
      __syncwarp();
#pragma unroll 1
      for (int part = 0; part < (nB ? 2 : 1); ++part)
        gyro_part(L, tile, part ? nA >> 2 : 0, part ? n >> 2 : nA >> 2, part ? lastB : lastA, slot->gidxG[part ? cur ^ 1 : cur], accG, ta, lane);
      if (nB) { ++c; cur ^= 1; endC = endB; }
      __syncwarp();
      pos += n;
    }
  }
  while (rounds-- > 0) { asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); }
}

}  // namespace tmi
}  // namespace icc
