// Residual + analytic Jacobian evaluation kernels (sm_90a), fused with the J^T J / J^T r reduction.
//
// Replaces, for every board-corner observation and every accelerometer / gyroscope sample in parallel, what the
// reference evaluates per residual block through ceres::DynamicAutoDiffCostFunction on CPU threads:
//   RSReprojectionCostFunctorSplit<6>::operator()   include/OpenCameraCalibrator/basalt_spline/ceres_calib_split_residuals.h:319-402
//   AccelerationCostFunctorSplit<6>::operator()     ...ceres_calib_split_residuals.h:52-93
//   GyroCostFunctorSplit<6,SO3,false>::operator()   ...ceres_calib_split_residuals.h:133-169
//   CeresSplineHelper<T,6>::evaluate_lie / evaluate ...ceres_spline_helper.h:101-220
// plus Ceres' J^T J assembly.  Jacobians are closed-form w.r.t. right-multiplicative increments of the six active
// SO(3) knots, the six R^3 knots, T_i_c (upsilon, omega), the line delay, gravity and the bias-spline knots, which is
// exactly autodiff x LieLocalParameterization of the reference (SURVEY.md §8(c)).
//
// Mapping to the machine: one WARP owns one work item (a camera frame / an IMU knot-interval cell), so the 6+6 knot
// window and the per-window quantities (log increments d_i, Jr^-1(d_i)) are staged ONCE in shared memory (16-byte
// vector loads of the padded knots); every lane evaluates one observation; each residual row [J | r] is written to a
// per-warp shared tile stored column-major (conflict-free) and the symmetric product [J|r]^T [J|r] is accumulated
// with FP64 tensor-core MMAs (mma.sync m8n8k4 f64: "tensor cores only where it is genuinely a contraction") into
// register fragments that persist across the whole work item; one atomic RED per tile entry then lands in the packed
// banded+bordered normal-equation buffer in HBM/L2.
#include "icc_camera.cuh"
#include "icc_kernels.h"
#include "icc_reduce.cuh"
#include "icc_spline_chain.cuh"
#include "icc_bearing_math.cuh"

#include <atomic>
#include <cstdlib>

namespace icc {

static std::atomic<int> g_launches{0};
int kernel_launch_count() { return g_launches.load(); }
void count_launch() { g_launches.fetch_add(1); }

namespace {

constexpr int WARPS = 4;
// tile columns of the CAM_INTRINSICS vision kernel (JAC == 2): [so3 | r3 | T_i_c | ld | MAX_INTR intrinsics | r] in 8-column blocks
constexpr int VIS_K_TILE_COLS = 8 * ((43 + MAX_INTR + 1 + 7) / 8);

ICC_D void mma_f64(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// acc += Jt^T Jt over rows [0, 4*nsteps) of the column-major tile; NB 8-column blocks; upper block triangle only.
template <int NB>
ICC_D void syrk_dmma(const double* __restrict__ Jt, int nsteps, double (&acc)[NB * (NB + 1) / 2][2]) {
  const int lane = threadIdx.x & 31;
  const double* base = Jt + (lane >> 2) * LDJ + (lane & 3);
  for (int s = 0; s < nsteps; ++s) {
    double f[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) f[b] = base[(8 * b) * LDJ + 4 * s];
    int idx = 0;
#pragma unroll
    for (int bi = 0; bi < NB; ++bi)
#pragma unroll
      for (int bj = bi; bj < NB; ++bj) { mma_f64(acc[idx], f[bi], f[bj]); ++idx; }
  }
}

ICC_D void ne_add(const DeviceProblem& P, int gi, int gj, double v) {
  const int lo = min(gi, gj), hi = max(gi, gj);
  double* dst;
  if (hi < P.nk) dst = P.ne + (int64_t)lo * P.ldb + (hi - lo);
  else if (lo < P.nk) dst = P.ne + P.ne_off_E + (int64_t)lo * P.nb + (hi - P.nk);
  else dst = P.ne + P.ne_off_C + (int64_t)(hi - P.nk) * P.nb + (lo - P.nk);
  atomicAdd(dst, v);
}

// Scatter the register fragments of one work item.  Local column `rescol` is the residual column:
// (I, rescol) -> gradient, (rescol, rescol) -> 2 * cost.
template <int NB>
ICC_D void flush_tile(const DeviceProblem& P, const int* gidx, int ncols, int rescol, double (&acc)[NB * (NB + 1) / 2][2]) {
  const int lane = threadIdx.x & 31;
  int idx = 0;
#pragma unroll
  for (int bi = 0; bi < NB; ++bi)
#pragma unroll
    for (int bj = bi; bj < NB; ++bj) {
      const int I = 8 * bi + (lane >> 2);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int J = 8 * bj + 2 * (lane & 3) + e;
        const double v = acc[idx][e];
        if (I < ncols && J < ncols && I <= J && v != 0.0) {
          if (J == rescol) {
            if (I == rescol) atomicAdd(P.ne + P.ne_off_cost, 0.5 * v);
            else { const int gi = gidx[I]; if (gi >= 0) atomicAdd(P.ne + P.ne_off_g + gi, v); }
          } else {
            const int gi = gidx[I], gj = gidx[J];
            if (gi >= 0 && gj >= 0) ne_add(P, gi, gj, v);
          }
        }
      }
      ++idx;
    }
}

// Stage the SO(3) window (6 knots -> 5 log increments and their Jr^-1) for one work item.
template <bool JAC>
ICC_D void stage_so3_window(WarpCtx* wc, const DeviceState& S, int s_so3, int lane) {
  if (lane < 6) { const double4 k = S.so3[s_so3 + lane]; wc->q[lane] = q4(k.x, k.y, k.z, k.w); }
  __syncwarp();
  if (lane < 5) stage_so3_increment<JAC>(wc, lane);
}

// ---------------------------------------------------------------------------------------------------------------
// Vision: rolling-shutter reprojection residuals.  Tile columns: [so3 0..17 | r3 18..35 | T_i_c 36..41 | ld 42 | r 43];
// JAC == 2 (CAM_INTRINSICS extension): [... | ld 42 | intrinsics 43..43+K-1 | r 43+K], K = parameter count of the model.
// TAN (JAC 0 / 1 only): the local tangent reprojection error against the corners' bearings (tangent_projection, icc_vision_rows.cuh).
// ---------------------------------------------------------------------------------------------------------------
template <int JAC, bool TAN = false>
__global__ void __launch_bounds__(WARPS * 32) vision_kernel(DeviceProblem P, DeviceState S, double* cost_out, double* res_out, double* reproj_out, TangentMeas T) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpCtx* wc = reinterpret_cast<WarpCtx*>(smem_raw) + warp;
  constexpr int NB = JAC == 2 ? VIS_K_TILE_COLS / 8 : 6, TILE_COLS = 8 * NB;
  double* Jt = reinterpret_cast<double*>(smem_raw + WARPS * sizeof(WarpCtx)) + warp * (TILE_COLS * LDJ);
  const int RES = JAC == 2 ? 43 + P.n_intr : 43, NCOL = RES + 1;
  double intr[MAX_INTR];
#pragma unroll
  for (int i = 0; i < MAX_INTR; ++i) intr[i] = S.glob[G_CAM_INTR + i];

  const Q4 q_ic = q4(S.glob[G_TIC + 0], S.glob[G_TIC + 1], S.glob[G_TIC + 2], S.glob[G_TIC + 3]);
  const V3 t_ic = v3(S.glob[G_TIC + 4], S.glob[G_TIC + 5], S.glob[G_TIC + 6]);
  const double ld = S.glob[G_LD];
  if (JAC) { for (int i = lane; i < TILE_COLS * LDJ; i += 32) Jt[i] = 0.0; }

  double cost_acc = 0.0, rp_sum = 0.0, rp_cnt = 0.0;
  for (int item = blockIdx.x * WARPS + warp; item < P.n_vwork; item += gridDim.x * WARPS) {
    const VisionWork wk = P.vwork[item];
    const int s_so3 = P.f_s_so3[wk.frame], s_r3 = P.f_s_r3[wk.frame];
    const double u_so3 = P.f_u_so3[wk.frame], u_r3 = P.f_u_r3[wk.frame];
    __syncwarp();
    if (lane < 6) { const double4 k = S.r3[s_r3 + lane]; wc->p[lane] = v3(k.x, k.y, k.z); }
    stage_so3_window<(JAC != 0)>(wc, S, s_so3, lane);
    if (JAC) {
      for (int c = lane; c < TILE_COLS; c += 32) {
        int g = -1;
        if (c < 18) { const int b = P.so3_col[s_so3 + c / 3]; g = b < 0 ? -1 : b + c % 3; }
        else if (c < 36) { const int b = P.r3_col[s_r3 + (c - 18) / 3]; g = b < 0 ? -1 : b + (c - 18) % 3; }
        else if (c < 42) g = P.col_tic < 0 ? -1 : P.col_tic + (c - 36);
        else if (c == 42) g = P.col_ld;
        else if (JAC == 2 && c < RES) g = P.col_ci < 0 ? -1 : P.col_ci + (c - 43);
        wc->gidx[c] = g;
      }
    }
    __syncwarp();
    double acc[NB * (NB + 1) / 2][2];
    if (JAC) {
#pragma unroll
      for (int i = 0; i < NB * (NB + 1) / 2; ++i) { acc[i][0] = 0.0; acc[i][1] = 0.0; }
    }
    for (int base = wk.c_begin; base < wk.c_end; base += 32) {
      const int c = base + lane;
      const bool act = c < wk.c_end;
      const int nact = min(32, wk.c_end - base);
      double r0 = 0.0, r1 = 0.0, y = 0.0;
      bool ok = false;
      Chain ch; Proj pr; ProjK pk; V3 qi = v3(0, 0, 0), pc = v3(0, 0, 0), tdot = v3(0, 0, 0);
      double cc[6];
      if (act) {
        const double2 ob = P.uv[c];
        y = ob.y;
        const double us = u_so3 + y * ld, ur = u_r3 + y * ld;   // residuals.h:344-346 (row time added to normalised u)
        build_chain(wc, us, ch);
        double dc[6];
        coeffs6(ur, cc, JAC ? dc : nullptr, nullptr);
        V3 t = v3(0, 0, 0);
#pragma unroll
        for (int j = 0; j < 6; ++j) { t = fma3(cc[j], wc->p[j], t); if (JAC) tdot = fma3(dc[j], wc->p[j], tdot); }
        const double4 X = P.board[P.pid[c]];
        qi = qrot_inv(ch.q, v3(X.x, X.y, X.z) - t);   // point in the IMU frame (board points are de-homogenised once, at upload)
        pc = qrot_inv(q_ic, qi - t_ic);                                // point in the camera frame
        if constexpr (TAN) {
          const bool b_ok = T.ok[c] != 0;
          pr = tangent_projection(T.bear[c], b_ok, T.s, pc);
          ok = pr.ok;
          if (ok) { r0 = pr.u; r1 = pr.v; } else if (!b_ok) { r0 = 0.0; r1 = 0.0; } else { r0 = 1e10; r1 = 1e10; }   // no bearing: zero residual
        } else {
          if (JAC == 2) pr = project_with_k(P.model, intr, pc, P.dispatch_fov != 0, &pk); else pr = project(P.model, intr, pc, P.dispatch_fov != 0);
          ok = pr.ok;
          if (ok) { r0 = pr.u - ob.x; r1 = pr.v - ob.y; } else { r0 = 1e10; r1 = 1e10; }   // residuals.h:391-398, cov = I
        }
        if (res_out) { res_out[2 * c] = r0; res_out[2 * c + 1] = r1; }
        if (!JAC) {
          cost_acc += 0.5 * (r0 * r0 + r1 * r1);
          if (reproj_out && r0 != 0.0 && r1 != 0.0) { rp_sum += sqrt(r0 * r0 + r1 * r1); rp_cnt += 1.0; }   // impl.h:1058-1064
        }
      }
      if (JAC) {
#pragma unroll 1
        for (int row = 0; row < 2; ++row) {
          if (act && ok) {
            const V3 Dp = v3(pr.J[3 * row], pr.J[3 * row + 1], pr.J[3 * row + 2]);
            const V3 m_q = qrot(q_ic, Dp);        // Dp R_ic^T as a covector
            const V3 m_th = cross(m_q, qi);       // m_q [qi]x
            const V3 m_t = qrot(ch.q, m_q);       // m_q R_wi^T
            const double du = so3_knot_row(wc, ch, m_th, Jt, lane, 1.0);
#pragma unroll
            for (int j = 0; j < 6; ++j) {
              Jt[(18 + 3 * j + 0) * LDJ + lane] = -cc[j] * m_t.x;
              Jt[(18 + 3 * j + 1) * LDJ + lane] = -cc[j] * m_t.y;
              Jt[(18 + 3 * j + 2) * LDJ + lane] = -cc[j] * m_t.z;
            }
            const V3 om = cross(Dp, pc);
            Jt[36 * LDJ + lane] = -Dp.x; Jt[37 * LDJ + lane] = -Dp.y; Jt[38 * LDJ + lane] = -Dp.z;
            Jt[39 * LDJ + lane] = om.x; Jt[40 * LDJ + lane] = om.y; Jt[41 * LDJ + lane] = om.z;
            Jt[42 * LDJ + lane] = y * (du - dot(m_t, tdot));
            if (JAC == 2) { for (int q = 0; q < P.n_intr; ++q) Jt[(43 + q) * LDJ + lane] = pk.Jk[jk_at(row, q)]; }
            Jt[RES * LDJ + lane] = row == 0 ? r0 : r1;
          } else {
            for (int k = 0; k < RES; ++k) Jt[k * LDJ + lane] = 0.0;
            Jt[RES * LDJ + lane] = act ? (row == 0 ? r0 : r1) : 0.0;
          }
          __syncwarp();
          syrk_dmma<NB>(Jt, (nact + 3) >> 2, acc);
          __syncwarp();
        }
      }
    }
    if (JAC) flush_tile<NB>(P, wc->gidx, NCOL, RES, acc);
  }
  if (!JAC) {
    cost_acc = warp_sum(cost_acc);
    if (lane == 0 && cost_out) atomicAdd(cost_out, cost_acc);
    if (reproj_out) { rp_sum = warp_sum(rp_sum); rp_cnt = warp_sum(rp_cnt); if (lane == 0) { atomicAdd(reproj_out, rp_sum); atomicAdd(reproj_out + 1, rp_cnt); } }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// IMU: accelerometer + gyroscope residuals of one knot-interval cell per warp.
//   accel tile columns: [so3 0..17 | r3 18..35 | g 36..38 | (ba 39..47) | (acc intr 48..53) | r]   NB = 5 / 7 / 7
//   gyro  tile columns: [so3 0..17 | (bg 18..26) | (gyr intr 27..35) | r]                          NB = 3 / 4 / 5
//   MODE 0 = biases fixed, 1 = bias knots free, 2 = widest: + IMU intrinsics (SplineOptimFlags::IMU_INTRINSICS) and the
//   time-offset increment (extension) as accel column 54 / gyro column 36
// ---------------------------------------------------------------------------------------------------------------
template <bool JAC, int MODE>
__global__ void __launch_bounds__(WARPS * 32) imu_kernel(DeviceProblem P, DeviceState S, double* cost_out, double* res_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr bool BIAS = MODE >= 1, INTR = MODE == 2;
  constexpr int NBA = BIAS ? 7 : 5, NBG = MODE == 0 ? 3 : MODE == 1 ? 4 : 5;
  constexpr int RESA = MODE == 0 ? 39 : MODE == 1 ? 48 : 55, NCOLA = RESA + 1, RESG = MODE == 0 ? 18 : MODE == 1 ? 27 : 37, NCOLG = RESG + 1;
  constexpr int TILE_COLS = 8 * NBA;
  WarpCtx* wc = reinterpret_cast<WarpCtx*>(smem_raw) + warp;
  double* Jt = reinterpret_cast<double*>(smem_raw + WARPS * sizeof(WarpCtx)) + warp * (TILE_COLS * LDJ);
  if (JAC) { for (int i = lane; i < TILE_COLS * LDJ; i += 32) Jt[i] = 0.0; }

  const double* ai = S.glob + G_ACC_INTR;
  const double* gi = S.glob + G_GYR_INTR;
  // misalignment * scale matrices (utils/types.h:226-246)
  const double Ma[9] = {ai[3], -ai[0] * ai[4], ai[1] * ai[5], 0.0, ai[4], -ai[2] * ai[5], 0.0, 0.0, ai[5]};
  const double Mg[9] = {gi[6], -gi[0] * gi[7], gi[1] * gi[8], gi[3] * gi[6], gi[7], -gi[2] * gi[8], -gi[4] * gi[6], gi[5] * gi[7], gi[8]};
  const V3 grav = v3(S.glob[G_GRAV], S.glob[G_GRAV + 1], S.glob[G_GRAV + 2]);
  const double idt2 = P.inv_r3_dt * P.inv_r3_dt;
  const double dto = S.glob[G_TOFF];   // time-offset increment [s] (0 unless the extension has been optimised)
  const double ba_rate = 1e9 / double(P.dt_ba_ns), bg_rate = 1e9 / double(P.dt_bg_ns);

  double cost_acc = 0.0;
  for (int item = blockIdx.x * WARPS + warp; item < P.n_iwork; item += gridDim.x * WARPS) {
    const ImuCell cell = P.iwork[item];
    __syncwarp();
    if (lane < 6) { const double4 k = S.r3[cell.s_r3 + lane]; wc->p[lane] = v3(k.x, k.y, k.z); }
    if (lane < 3) { const double4 a = S.ba[cell.s_ba + lane]; wc->ba[lane] = v3(a.x, a.y, a.z); const double4 g = S.bg[cell.s_bg + lane]; wc->bg[lane] = v3(g.x, g.y, g.z); }
    stage_so3_window<JAC>(wc, S, cell.s_so3, lane);
    if (JAC) {
      for (int c = lane; c < 64; c += 32) {
        int g = -1;
        if (c < 18) { const int b = P.so3_col[cell.s_so3 + c / 3]; g = b < 0 ? -1 : b + c % 3; }
        else if (c < 36) { const int b = P.r3_col[cell.s_r3 + (c - 18) / 3]; g = b < 0 ? -1 : b + (c - 18) % 3; }
        else if (c < 39) g = P.col_g < 0 ? -1 : P.col_g + (c - 36);
        else if (BIAS && c < 48) { const int b = P.ba_col[cell.s_ba + (c - 39) / 3]; g = b < 0 ? -1 : b + (c - 39) % 3; }
        else if (INTR && c < 54) g = P.col_ai < 0 ? -1 : P.col_ai + (c - 48);
        else if (INTR && c == 54) g = P.col_to;
        wc->gidx[c] = g;
      }
      for (int c = lane; c < 40; c += 32) {
        int g = -1;
        if (c < 18) { const int b = P.so3_col[cell.s_so3 + c / 3]; g = b < 0 ? -1 : b + c % 3; }
        else if (BIAS && c < 27) { const int b = P.bg_col[cell.s_bg + (c - 18) / 3]; g = b < 0 ? -1 : b + (c - 18) % 3; }
        else if (INTR && c < 36) g = P.col_gi < 0 ? -1 : P.col_gi + (c - 27);
        else if (INTR && c == 36) g = P.col_to;
        wc->gidx2[c] = g;
      }
    }
    __syncwarp();
    double accA[NBA * (NBA + 1) / 2][2], accG[NBG * (NBG + 1) / 2][2];
    if (JAC) {
#pragma unroll
      for (int i = 0; i < NBA * (NBA + 1) / 2; ++i) { accA[i][0] = 0.0; accA[i][1] = 0.0; }
#pragma unroll
      for (int i = 0; i < NBG * (NBG + 1) / 2; ++i) { accG[i][0] = 0.0; accG[i][1] = 0.0; }
    }
    for (int base = cell.i_begin; base < cell.i_end; base += 32) {
      const int i = base + lane;
      const bool act = i < cell.i_end;
      const int nact = min(32, cell.i_end - base);
      const int nsteps = (nact + 3) >> 2;
      Chain ch;
      double ra[3] = {0, 0, 0}, rg[3] = {0, 0, 0};
      double ddc[6], cba[3], cbg[3];
      V3 h = v3(0, 0, 0), va = v3(0, 0, 0), vg = v3(0, 0, 0);   // va / vg: raw readings minus bias
      V3 dacc = v3(0, 0, 0), dgyr = v3(0, 0, 0);                // d residual / d time offset (unweighted), MODE 2 only
      if (act) {
        const int64_t st = P.imu_t_ns[i];
        // CalcTimes (impl.h:763-788): u = (st % dt) / dt with the segment index known from the cell
        const double u_so3 = double(st - (int64_t)cell.s_so3 * P.dt_so3_ns) / double(P.dt_so3_ns) + dto * P.inv_so3_dt;
        const double u_r3 = double(st - (int64_t)cell.s_r3 * P.dt_r3_ns) / double(P.dt_r3_ns) + dto * P.inv_r3_dt;
        const double u_ba = double(st - (int64_t)cell.s_ba * P.dt_ba_ns) / double(P.dt_ba_ns) + dto * ba_rate;
        const double u_bg = double(st - (int64_t)cell.s_bg * P.dt_bg_ns) / double(P.dt_bg_ns) + dto * bg_rate;
        build_chain(wc, u_so3, ch);
        double cdum[6];
        coeffs6(u_r3, cdum, nullptr, ddc);
        coeffs3(u_ba, cba); coeffs3(u_bg, cbg);
        // accelerometer residual (residuals.h:52-93)
        V3 aw = v3(0, 0, 0);
#pragma unroll
        for (int j = 0; j < 6; ++j) aw = fma3(ddc[j] * idt2, wc->p[j], aw);
        h = qrot_inv(ch.q, aw + grav);
        V3 bacc = v3(0, 0, 0), bgyr = v3(0, 0, 0);
#pragma unroll
        for (int k = 0; k < 3; ++k) { bacc = fma3(cba[k], wc->ba[k], bacc); bgyr = fma3(cbg[k], wc->bg[k], bgyr); }
        const V3 a_raw = v3(P.imu_acc[3 * i], P.imu_acc[3 * i + 1], P.imu_acc[3 * i + 2]) - bacc;
        const V3 g_raw = v3(P.imu_gyr[3 * i], P.imu_gyr[3 * i + 1], P.imu_gyr[3 * i + 2]) - bgyr;
        va = a_raw; vg = g_raw;
        ra[0] = P.w_acc * (h.x - (Ma[0] * a_raw.x + Ma[1] * a_raw.y + Ma[2] * a_raw.z));
        ra[1] = P.w_acc * (h.y - (Ma[3] * a_raw.x + Ma[4] * a_raw.y + Ma[5] * a_raw.z));
        ra[2] = P.w_acc * (h.z - (Ma[6] * a_raw.x + Ma[7] * a_raw.y + Ma[8] * a_raw.z));
        // gyroscope residual (residuals.h:133-169): body velocity recursion (spline_helper.h:159-164)
        V3 om = v3(0, 0, 0);
#pragma unroll
        for (int k = 0; k < 5; ++k) om = qrot_inv(ch.A[k], om) + (ch.dlam[k] * P.inv_so3_dt) * wc->d[k];
        rg[0] = P.w_gyr * (om.x - (Mg[0] * g_raw.x + Mg[1] * g_raw.y + Mg[2] * g_raw.z));
        rg[1] = P.w_gyr * (om.y - (Mg[3] * g_raw.x + Mg[4] * g_raw.y + Mg[5] * g_raw.z));
        rg[2] = P.w_gyr * (om.z - (Mg[6] * g_raw.x + Mg[7] * g_raw.y + Mg[8] * g_raw.z));
        if (JAC && INTR) {
          // d/d(time offset): accel  d(R^T v)/dt = h x omega + R^T jerk (+ M_a db_a/dt);  gyro  d omega/dt = body angular
          // acceleration, recursion of CeresSplineHelper::evaluate_lie (ceres_spline_helper.h:166-170)  (+ M_g db_g/dt)
          double dddc[6], ddlam[5], dcba[3], dcbg[3];
          coeffs6_ddd(u_r3, dddc); cum_coeffs6_dd(u_so3, ddlam); coeffs3_d(u_ba, dcba); coeffs3_d(u_bg, dcbg);
          V3 jerk = v3(0, 0, 0);
#pragma unroll
          for (int j = 0; j < 6; ++j) jerk = fma3(dddc[j] * idt2 * P.inv_r3_dt, wc->p[j], jerk);
          V3 dba = v3(0, 0, 0), dbg = v3(0, 0, 0);
#pragma unroll
          for (int k = 0; k < 3; ++k) { dba = fma3(dcba[k] * ba_rate, wc->ba[k], dba); dbg = fma3(dcbg[k] * bg_rate, wc->bg[k], dbg); }
          V3 rv = v3(0, 0, 0), racc = v3(0, 0, 0);
#pragma unroll
          for (int k = 0; k < 5; ++k) {
            const V3 cur = (ch.dlam[k] * P.inv_so3_dt) * wc->d[k];
            rv = qrot_inv(ch.A[k], rv) + cur;
            racc = qrot_inv(ch.A[k], racc) + (ddlam[k] * P.inv_so3_dt * P.inv_so3_dt) * wc->d[k] + cross(rv, cur);
          }
          const V3 t1 = cross(h, om) + qrot_inv(ch.q, jerk);
          dacc = v3(t1.x + Ma[0] * dba.x + Ma[1] * dba.y + Ma[2] * dba.z, t1.y + Ma[3] * dba.x + Ma[4] * dba.y + Ma[5] * dba.z, t1.z + Ma[6] * dba.x + Ma[7] * dba.y + Ma[8] * dba.z);
          dgyr = v3(racc.x + Mg[0] * dbg.x + Mg[1] * dbg.y + Mg[2] * dbg.z, racc.y + Mg[3] * dbg.x + Mg[4] * dbg.y + Mg[5] * dbg.z, racc.z + Mg[6] * dbg.x + Mg[7] * dbg.y + Mg[8] * dbg.z);
        }
        if (res_out) {
#pragma unroll
          for (int k = 0; k < 3; ++k) { res_out[P.n_res_vis + 3 * i + k] = ra[k]; res_out[P.n_res_vis + P.n_res_acc + 3 * i + k] = rg[k]; }
        }
        if (!JAC) cost_acc += 0.5 * (ra[0] * ra[0] + ra[1] * ra[1] + ra[2] * ra[2] + rg[0] * rg[0] + rg[1] * rg[1] + rg[2] * rg[2]);
      }
      if (JAC) {
        // ---- accelerometer rows -----------------------------------------------------------------------------
#pragma unroll 1
        for (int k = 0; k < 3; ++k) {
          if (act) {
            const V3 ek = v3(k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0);
            const V3 m_th = cross(ek, h);              // e_k^T [h]x
            const V3 m_t = qrot(ch.q, ek);             // e_k^T R_wi^T
            so3_knot_row(wc, ch, m_th, Jt, lane, P.w_acc);
#pragma unroll
            for (int j = 0; j < 6; ++j) {
              const double s = P.w_acc * ddc[j] * idt2;
              Jt[(18 + 3 * j + 0) * LDJ + lane] = s * m_t.x; Jt[(18 + 3 * j + 1) * LDJ + lane] = s * m_t.y; Jt[(18 + 3 * j + 2) * LDJ + lane] = s * m_t.z;
            }
            Jt[36 * LDJ + lane] = P.w_acc * m_t.x; Jt[37 * LDJ + lane] = P.w_acc * m_t.y; Jt[38 * LDJ + lane] = P.w_acc * m_t.z;
            if (BIAS) {
#pragma unroll
              for (int j = 0; j < 3; ++j) {
                const double s = P.w_acc * cba[j];
                Jt[(39 + 3 * j + 0) * LDJ + lane] = s * Ma[3 * k + 0]; Jt[(39 + 3 * j + 1) * LDJ + lane] = s * Ma[3 * k + 1]; Jt[(39 + 3 * j + 2) * LDJ + lane] = s * Ma[3 * k + 2];
              }
            }
            if (INTR) {   // d(-M_a v)/d[misYZ, misZY, misZX, sX, sY, sZ], M_a = [[sX, -yz sY, zy sZ],[0, sY, -zx sZ],[0, 0, sZ]]
              const double d[6] = {k == 0 ? ai[4] * va.y : 0.0, k == 0 ? -ai[5] * va.z : 0.0, k == 1 ? ai[5] * va.z : 0.0,
                                   k == 0 ? -va.x : 0.0, k == 0 ? ai[0] * va.y : (k == 1 ? -va.y : 0.0), k == 0 ? -ai[1] * va.z : (k == 1 ? ai[2] * va.z : -va.z)};
#pragma unroll
              for (int q = 0; q < 6; ++q) Jt[(48 + q) * LDJ + lane] = P.w_acc * d[q];
              Jt[54 * LDJ + lane] = P.w_acc * (k == 0 ? dacc.x : k == 1 ? dacc.y : dacc.z);
            }
            Jt[RESA * LDJ + lane] = ra[k];
          } else {
            for (int c = 0; c < NCOLA; ++c) Jt[c * LDJ + lane] = 0.0;
          }
          __syncwarp();
          syrk_dmma<NBA>(Jt, nsteps, accA);
          __syncwarp();
        }
        // ---- gyroscope rows ------------------------------------------------------------------------------------
#pragma unroll 1
        for (int k = 0; k < 3; ++k) {
          if (act) {
            // d omega_k / d eps_j = y_j Jr^-1_j - Jr^-1_{j+1} y_{j+1},  y_i = lam_i ((w_i x s_i) Jr(phi_i)) + lam'_i w_i
            // s_i = A_i^T omega_{i-1} needs the forward recursion; recompute it backwards-compatible: store s_i first.
            V3 s[5];
            {
              V3 om = v3(0, 0, 0);
#pragma unroll
              for (int i2 = 0; i2 < 5; ++i2) { s[i2] = qrot_inv(ch.A[i2], om); om = s[i2] + (ch.dlam[i2] * P.inv_so3_dt) * wc->d[i2]; }
            }
            V3 w = v3(k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0);
            V3 z_next = v3(0, 0, 0);
#pragma unroll
            for (int i2 = 4; i2 >= 0; --i2) {
              const V3 yv = lam_row_jr(cross(w, s[i2]), wc->dh[i2], ch.lam[i2], ch.c1[i2], ch.c2[i2]) + (ch.dlam[i2] * P.inv_so3_dt) * w;
              const V3 up = mulT(wc->jri[i2], yv) - z_next;
              Jt[(3 * (i2 + 1) + 0) * LDJ + lane] = P.w_gyr * up.x; Jt[(3 * (i2 + 1) + 1) * LDJ + lane] = P.w_gyr * up.y; Jt[(3 * (i2 + 1) + 2) * LDJ + lane] = P.w_gyr * up.z;
              z_next = mul(wc->jri[i2], yv);
              w = qrot(ch.A[i2], w);
            }
            Jt[0 * LDJ + lane] = -P.w_gyr * z_next.x; Jt[1 * LDJ + lane] = -P.w_gyr * z_next.y; Jt[2 * LDJ + lane] = -P.w_gyr * z_next.z;
            if (BIAS) {
#pragma unroll
              for (int j = 0; j < 3; ++j) {
                const double sc = P.w_gyr * cbg[j];
                Jt[(18 + 3 * j + 0) * LDJ + lane] = sc * Mg[3 * k + 0]; Jt[(18 + 3 * j + 1) * LDJ + lane] = sc * Mg[3 * k + 1]; Jt[(18 + 3 * j + 2) * LDJ + lane] = sc * Mg[3 * k + 2];
              }
            }
            if (INTR) {   // d(-M_g v)/d[misYZ, misZY, misZX, misXZ, misXY, misYX, sX, sY, sZ]
              double d[9];
              if (k == 0) { d[0] = gi[7] * vg.y; d[1] = -gi[8] * vg.z; d[2] = 0; d[3] = 0; d[4] = 0; d[5] = 0; d[6] = -vg.x; d[7] = gi[0] * vg.y; d[8] = -gi[1] * vg.z; }
              else if (k == 1) { d[0] = 0; d[1] = 0; d[2] = gi[8] * vg.z; d[3] = -gi[6] * vg.x; d[4] = 0; d[5] = 0; d[6] = -gi[3] * vg.x; d[7] = -vg.y; d[8] = gi[2] * vg.z; }
              else { d[0] = 0; d[1] = 0; d[2] = 0; d[3] = 0; d[4] = gi[6] * vg.x; d[5] = -gi[7] * vg.y; d[6] = gi[4] * vg.x; d[7] = -gi[5] * vg.y; d[8] = -vg.z; }
#pragma unroll
              for (int q = 0; q < 9; ++q) Jt[(27 + q) * LDJ + lane] = P.w_gyr * d[q];
              Jt[36 * LDJ + lane] = P.w_gyr * (k == 0 ? dgyr.x : k == 1 ? dgyr.y : dgyr.z);
            }
            Jt[RESG * LDJ + lane] = rg[k];
            for (int c = NCOLG; c < 8 * NBG; ++c) Jt[c * LDJ + lane] = 0.0;
          } else {
            for (int c = 0; c < 8 * NBG; ++c) Jt[c * LDJ + lane] = 0.0;
          }
          __syncwarp();
          syrk_dmma<NBG>(Jt, nsteps, accG);
          __syncwarp();
        }
        // the accelerometer layout is wider than the gyroscope one: clear what the gyro rows overwrote beyond their own
        // columns is unnecessary (accel rewrites all its columns), but the accel PAD columns must stay zero: they are never written.
      }
    }
    if (JAC) {
      flush_tile<NBA>(P, wc->gidx, NCOLA, RESA, accA);
      flush_tile<NBG>(P, wc->gidx2, NCOLG, RESG, accG);
    }
  }
  if (!JAC) {
    cost_acc = warp_sum(cost_acc);
    if (lane == 0 && cost_out) atomicAdd(cost_out, cost_acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Trajectory getters (impl.h:898-991,1180-1234), one thread per timestamp.
// ---------------------------------------------------------------------------------------------------------------
__device__ bool calc_times_dev(int64_t t_ns, int64_t start_ns, int64_t dt_ns, int nr_knots, int N, double& u, int& s) {
  const int64_t st = t_ns - start_ns;
  if (st < 0) return false;
  const int64_t sl = st / dt_ns;
  if (sl + N > (int64_t)nr_knots) return false;
  s = (int)sl; u = double(st % dt_ns) / double(dt_ns);
  return true;
}

__global__ void trajectory_kernel(DeviceProblem P, DeviceState S, int n, const int64_t* t_ns, int64_t start_ns, double* gyro, double* accel, double* bg,
                                  double* ba, double* pose_q, double* pose_p, int* valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double u_so3 = 0, u_r3 = 0, u_b = 0; int s_so3 = 0, s_r3 = 0, s_b = 0;
  const bool ok_so3 = calc_times_dev(t_ns[i], start_ns, P.dt_so3_ns, P.n_so3, SPLINE_N, u_so3, s_so3);
  const bool ok_r3 = calc_times_dev(t_ns[i], start_ns, P.dt_r3_ns, P.n_r3, SPLINE_N, u_r3, s_r3);
  if (valid) valid[i] = ok_so3 && ok_r3;
  Q4 R = q4(0, 0, 0, 1); V3 om = v3(0, 0, 0);
  if (ok_so3) {
    double lam[5], dlam[5];
    cum_coeffs6(u_so3, lam, dlam);
    double4 k0 = S.so3[s_so3];
    Q4 prev = q4(k0.x, k0.y, k0.z, k0.w);
    R = prev;
    for (int k = 0; k < 5; ++k) {
      const double4 kn = S.so3[s_so3 + k + 1];
      const Q4 next = q4(kn.x, kn.y, kn.z, kn.w);
      const V3 d = so3_log(qmul(qconj(prev), next));
      const Q4 A = so3_exp(lam[k] * d);
      R = qmul(R, A);
      om = qrot_inv(A, om) + (dlam[k] * P.inv_so3_dt) * d;
      prev = next;
    }
  }
  if (gyro && ok_so3) { gyro[3 * i] = om.x; gyro[3 * i + 1] = om.y; gyro[3 * i + 2] = om.z; }
  if (ok_so3 && ok_r3) {
    double c[6], ddc[6];
    coeffs6(u_r3, c, nullptr, ddc);
    V3 p = v3(0, 0, 0), a = v3(0, 0, 0);
    for (int k = 0; k < 6; ++k) { const double4 kk = S.r3[s_r3 + k]; const V3 kv = v3(kk.x, kk.y, kk.z); p = fma3(c[k], kv, p); a = fma3(ddc[k] * P.inv_r3_dt * P.inv_r3_dt, kv, a); }
    if (accel) { const V3 h = qrot_inv(R, a + v3(S.glob[G_GRAV], S.glob[G_GRAV + 1], S.glob[G_GRAV + 2])); accel[3 * i] = h.x; accel[3 * i + 1] = h.y; accel[3 * i + 2] = h.z; }
    if (pose_q) { pose_q[4 * i] = R.x; pose_q[4 * i + 1] = R.y; pose_q[4 * i + 2] = R.z; pose_q[4 * i + 3] = R.w; }
    if (pose_p) { pose_p[3 * i] = p.x; pose_p[3 * i + 1] = p.y; pose_p[3 * i + 2] = p.z; }
  }
  if (bg) {
    V3 b = v3(0, 0, 0);
    if (calc_times_dev(t_ns[i], start_ns, P.dt_bg_ns, P.n_bg, BIAS_N, u_b, s_b)) { double c[3]; coeffs3(u_b, c); for (int k = 0; k < 3; ++k) { const double4 kk = S.bg[s_b + k]; b = fma3(c[k], v3(kk.x, kk.y, kk.z), b); } }
    bg[3 * i] = b.x; bg[3 * i + 1] = b.y; bg[3 * i + 2] = b.z;
  }
  if (ba) {
    V3 b = v3(0, 0, 0);
    if (calc_times_dev(t_ns[i], start_ns, P.dt_ba_ns, P.n_ba, BIAS_N, u_b, s_b)) { double c[3]; coeffs3(u_b, c); for (int k = 0; k < 3; ++k) { const double4 kk = S.ba[s_b + k]; b = fma3(c[k], v3(kk.x, kk.y, kk.z), b); } }
    ba[3 * i] = b.x; ba[3 * i + 1] = b.y; ba[3 * i + 2] = b.z;
  }
}

template <typename K>
int set_smem(K kernel, size_t bytes) { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess ? 0 : 1; }

int grid_for(int n_items, int sm_count) { const int ctas = (n_items + WARPS - 1) / WARPS; return ctas < 1 ? 1 : (ctas > sm_count * 8 ? sm_count * 8 : ctas); }

}  // namespace

int launch_eval(const DeviceProblem& P_in, const DeviceState& S, bool with_jacobian, double* cost_out, double* residuals_out, double* reproj_out, cudaStream_t st_main, const EvalAux* aux, const TangentMeas* tan) {
  DeviceProblem P = P_in;
  if (S.board) P.board = S.board;   // the board points belong to the state (parameter blocks under SplineOptimFlags::POINTS)
  static int sm_count = 0;
  if (!sm_count) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev); if (sm_count <= 0) sm_count = 132; }
  const size_t sm_vis = WARPS * sizeof(WarpCtx) + WARPS * 48 * LDJ * sizeof(double);
  const size_t sm_vis_k = WARPS * sizeof(WarpCtx) + WARPS * VIS_K_TILE_COLS * LDJ * sizeof(double);
  const size_t sm_imu_nb = WARPS * sizeof(WarpCtx) + WARPS * 40 * LDJ * sizeof(double);
  const size_t sm_imu_b = WARPS * sizeof(WarpCtx) + WARPS * 56 * LDJ * sizeof(double);
  const size_t sm_cost = WARPS * sizeof(WarpCtx);   // the cost-only kernels never touch a tile: more CTAs per SM
  static bool attr_done = false;
  if (!attr_done) {
    int e = 0;
    e |= set_smem(vision_kernel<1>, sm_vis); e |= set_smem(vision_kernel<0>, sm_vis); e |= set_smem(vision_kernel<2>, sm_vis_k);
    e |= set_smem(vision_kernel<1, true>, sm_vis); e |= set_smem(vision_kernel<0, true>, sm_vis);
    e |= set_smem(imu_kernel<true, 0>, sm_imu_nb); e |= set_smem(imu_kernel<false, 0>, sm_imu_nb);
    e |= set_smem(imu_kernel<true, 1>, sm_imu_b); e |= set_smem(imu_kernel<false, 1>, sm_imu_b); e |= set_smem(imu_kernel<true, 2>, sm_imu_b);
    if (e) return 1;
    attr_done = true;
  }
  // Jacobian evaluations of the standard column sets run as items of the persistent shared-memory-parking kernel (icc_eval_tmem.cu), which owns
  // every SM (one CTA each); whatever is not eligible (camera intrinsics / bias knots / IMU intrinsics free) follows on the same stream.
  const bool legacy_vision = getenv("ICC_VISION_LEGACY") != nullptr;   // A/B switch for profiling only (read per call)
  // size test: the persistent kernel pays off once every warp has a few chunks (BASELINE config 4 on 132 SMs: 12.8 vision / 3.1 IMU chunks per warp);
  // below that the one-warp-per-frame / per-cell kernels finish sooner and run side by side
  const int tm_vwarps = sm_count * eval_tmem_warps(false), tm_iwarps = sm_count * eval_tmem_warps(true);
  const bool tmem_vision = with_jacobian && !P.cam_intr_active && P.n_vitems > 0 && P.rolling && !legacy_vision && (P.n_vchunks >= 3 * tm_vwarps || getenv("ICC_TMEM_ALWAYS"));
  const bool legacy_imu = getenv("ICC_IMU_LEGACY") != nullptr;
  const bool tmem_imu = with_jacobian && !P.bias_active && !P.intr_active && P.n_iitems > 0 && P.n_iwork > 0 && !legacy_imu && (2 * P.n_ichunks >= 3 * tm_iwarps || getenv("ICC_TMEM_ALWAYS"));
  const bool fork = aux && P.n_vwork > 0 && P.rolling && P.n_iwork > 0 && !tmem_vision && !tmem_imu;
  cudaStream_t st = st_main;
  if (fork) { cudaEventRecord(aux->fork, st_main); cudaStreamWaitEvent(aux->stream, aux->fork, 0); }
  if (tmem_vision || tmem_imu) {   // one persistent launch for every item type that is eligible
    DeviceProblem Q = P;
    if (!tmem_vision) Q.n_vitems = 0;
    if (!tmem_imu) Q.n_iitems = 0;
    if (launch_eval_tmem(Q, S, residuals_out, sm_count, st, tan)) return 1;
  }
  if (tmem_vision) {
  } else if (P.n_vwork > 0 && P.rolling) {
    const int grid = grid_for(P.n_vwork, sm_count);
    const TangentMeas T = tan ? *tan : TangentMeas{nullptr, nullptr, 0.0};
    if (tan) {   // (icc_api.cu refuses CAM_INTRINSICS in tangent mode)
      if (with_jacobian) vision_kernel<1, true><<<grid, WARPS * 32, sm_vis, st>>>(P, S, cost_out, residuals_out, reproj_out, T);
      else vision_kernel<0, true><<<grid, WARPS * 32, sm_cost, st>>>(P, S, cost_out, residuals_out, reproj_out, T);
    } else if (with_jacobian && P.cam_intr_active) vision_kernel<2><<<grid, WARPS * 32, sm_vis_k, st>>>(P, S, cost_out, residuals_out, reproj_out, T);
    else if (with_jacobian) vision_kernel<1><<<grid, WARPS * 32, sm_vis, st>>>(P, S, cost_out, residuals_out, reproj_out, T);
    else vision_kernel<0><<<grid, WARPS * 32, sm_cost, st>>>(P, S, cost_out, residuals_out, reproj_out, T);
    count_launch();
  }
  if (tmem_imu) {
  } else if (P.n_iwork > 0) {
    if (fork) st = aux->stream;
    const int grid = grid_for(P.n_iwork, sm_count);
    if (P.bias_active || P.intr_active) {
      if (with_jacobian && P.intr_active) imu_kernel<true, 2><<<grid, WARPS * 32, sm_imu_b, st>>>(P, S, cost_out, residuals_out);
      else if (with_jacobian) imu_kernel<true, 1><<<grid, WARPS * 32, sm_imu_b, st>>>(P, S, cost_out, residuals_out);
      else imu_kernel<false, 1><<<grid, WARPS * 32, sm_cost, st>>>(P, S, cost_out, residuals_out);
    } else {
      if (with_jacobian) imu_kernel<true, 0><<<grid, WARPS * 32, sm_imu_nb, st>>>(P, S, cost_out, residuals_out);
      else imu_kernel<false, 0><<<grid, WARPS * 32, sm_cost, st>>>(P, S, cost_out, residuals_out);
    }
    count_launch();
  }
  if (fork) { cudaEventRecord(aux->join, aux->stream); cudaStreamWaitEvent(st_main, aux->join, 0); }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

void launch_eval_trajectory(const DeviceProblem& P, const DeviceState& S, int n, const int64_t* t_ns, int64_t start_ns, double* gyro, double* accel,
                            double* bg, double* ba, double* pose_q, double* pose_p, int* valid, cudaStream_t st) {
  if (n <= 0) return;
  trajectory_kernel<<<(n + 127) / 128, 128, 0, st>>>(P, S, n, t_ns, start_ns, gyro, accel, bg, ba, pose_q, pose_p, valid);
  count_launch();
}

}  // namespace icc
