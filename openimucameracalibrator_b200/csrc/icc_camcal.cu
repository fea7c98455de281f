// Camera intrinsic calibration (sm_90a): bundle adjustment of every view pose + ONE shared intrinsic vector (SURVEY.md §8(f) row f4).
//
// Replaces what the reference delegates to theia::BundleAdjustViews (Ceres, DENSE/SPARSE_SCHUR, autodiff, CPU threads) in
//   CameraCalibrator::RunCalibration            src/core/camera_calibrator.cc:131-219   (three stages, Huber 1.345)
//   utils::GetReprojErrorOfView                 src/utils/utils.cc:163-177              (per-view mean reprojection error)
// with the residual of theia::ReprojectionError (external): r = CameraToPixelCoordinates(intr, R_cw (X - c)) - feature.
//
// Mapping to the machine.  The normal equations are an arrow: 6x6 pose blocks on the diagonal, a border of <= MAX_INTR (13) intrinsics.
//   camcal_accumulate_kernel : one WARP per view.  Each lane evaluates one corner (projection + closed-form 2x3 and 2xMAX_INTR
//       Jacobians of icc_camera.cuh, Huber weight) and writes its weighted rows [J_pose | J_intr | r] (17 columns, padded to three
//       8-column blocks) into the warp's shared-memory tile -- x rows, then y rows; each half is folded into the symmetric product
//       with FP64 tensor-core MMAs (mma.sync m8n8k4: 6 block products per 4 rows, the accumulator fragments stay in registers for
//       the whole view), so J^T J, J^T r and r^T r come out of one contraction.  The view's 17x17 block goes to HBM, its intrinsics
//       part is summed into the global system with RED.ADD.F64.
//   camcal_reduce_kernel     : one thread per view: damped 6x6 Cholesky, Y = A^-1 [H_pk | g_p], Schur complement of the view
//       onto the intrinsics, summed over the CTA through shared memory and added to the reduced MAX_INTR x MAX_INTR system.
//   camcal_solve_kernel      : the reduced system (<= MAX_INTR unknowns) by Cholesky, intrinsics step, candidate intrinsics.
//   camcal_update_kernel     : back-substitution of every view's pose step, candidate poses, step / model-decrease sums.
// The host only sequences these launches and applies Ceres' trust-region logic to eight scalars per iteration (calibrate_camera below).
#include "icc_camera.cuh"
#include "icc_host.h"
#include "icc_reduce.cuh"
#include "icc_rolling_shutter_math.cuh"
#include "icc_small_linalg.cuh"
#include "icc_trust_region.cuh"

#include <chrono>
#include <cmath>
#include <unordered_map>

namespace icc {

// Column order of a view's [J | r] rows: 0-2 rotation increment, 3-5 camera centre, 6.. intrinsics (Theia order, MAX_INTR columns), residual.
constexpr int CC_RES = 6 + MAX_INTR, CC_COLS = CC_RES + 1, CC_PACK = CC_COLS * (CC_COLS + 1) / 2;   // packed upper triangle
constexpr int CC_Y = 6 * (MAX_INTR + 1);                                                           // Y = A^-1 [H_pk | g_p] (6 x (MAX_INTR + 1))
// the intrinsics' Schur complement: the packed upper triangle of the reduced system, then its gradient
constexpr int CC_RED_G = MAX_INTR * (MAX_INTR + 1) / 2, CC_RED = CC_RED_G + MAX_INTR;
enum { CC_CAND_COST = 0, CC_G_DELTA = 1, CC_D_DELTA = 2, CC_STEP_SQ = 3, CC_X_SQ = 4, CC_FAIL = 5, CC_GRAD_MAX = 6, CC_X_COST = 7, CC_SCAL_COUNT = 8 };
struct CamCalProblem {
  int model, n_points, n_active, pose_free;
  unsigned intr_mask;          // bit i set = intrinsic i is optimised in this stage
  double huber;                // loss width (camera_calibrator.cc:143)
  const double4* board; const int* f_off; const int* pid; const double2* uv;
  const int* active;           // indices of the views that take part (n_active)
};
struct CamCalState { double* q; double* c; double* k; };   // R_cw as (x,y,z,w) per view, camera centre per view, MAX_INTR intrinsics
struct CamCalRs { const double* vel; double line_delay; };  // rolling shutter: (w, u) per view (6 doubles), line delay [s]; vel == nullptr: global

namespace {

ICC_HD int pk(int i, int j) { return i * CC_COLS - i * (i - 1) / 2 + (j - i); }              // packed upper triangle of a view's block, i <= j
ICC_HD int pkr(int a, int b) { return a * MAX_INTR - a * (a - 1) / 2 + (b - a); }             // packed upper triangle of the reduced system

ICC_D void atomic_max_nonneg(double* addr, double v) {   // v >= 0: the bit patterns of non-negative doubles order like integers
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

ICC_D void mma_f64(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
constexpr int CC_NB = 3, CC_TCOLS = 8 * CC_NB, CC_NACC = CC_NB * (CC_NB + 1) / 2;
constexpr int LDT = 36;   // tile rows per column (32 + 4 pad: stride = 4 mod 16 => conflict-free fragment loads)

// acc += T^T T over rows [0, 4 nsteps) of the column-major tile (upper block triangle of the 3 x 3 blocks of 8 columns)
ICC_D void syrk_tile(const double* __restrict__ T, int nsteps, double (&acc)[CC_NACC][2]) {
  const int lane = threadIdx.x & 31;
  const double* base = T + (lane >> 2) * LDT + (lane & 3);
  for (int s = 0; s < nsteps; ++s) {
    double f[CC_NB];
#pragma unroll
    for (int b = 0; b < CC_NB; ++b) f[b] = base[(8 * b) * LDT + 4 * s];
    int idx = 0;
#pragma unroll
    for (int bi = 0; bi < CC_NB; ++bi)
#pragma unroll
      for (int bj = bi; bj < CC_NB; ++bj) { mma_f64(acc[idx], f[bi], f[bj]); ++idx; }
  }
}

// RS: rolling shutter (icc_set_camcal_rolling_shutter): corner c is predicted at its row time uv[c].y * rs.line_delay from P(tau) with the
// view's velocities rs.vel[6 v .. 6 v + 5] (rs_camera_residual); RS = false is the global-shutter kernel, and never reads rs.
template <bool JAC, bool RS>
__global__ void __launch_bounds__(128) camcal_accumulate_kernel(CamCalProblem Q, CamCalState S, double* __restrict__ blocks, double* __restrict__ sys,
                                                               double* __restrict__ cost_out, double* __restrict__ view_err, CamCalRs rs) {
  __shared__ double tile_all[JAC ? 4 * CC_TCOLS * LDT : 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = blockIdx.x * 4 + warp;
  if (slot >= Q.n_active) return;
  double* tile = tile_all + (JAC ? warp * CC_TCOLS * LDT : 0);
  if (JAC) { for (int i = lane; i < CC_TCOLS * LDT; i += 32) tile[i] = 0.0; __syncwarp(); }   // the padding columns past CC_COLS stay zero
  const int v = Q.active[slot];
  const int c0 = Q.f_off[v], c1 = Q.f_off[v + 1];
  const Q4 q = q4(S.q[4 * v], S.q[4 * v + 1], S.q[4 * v + 2], S.q[4 * v + 3]);
  const V3 cc = v3(S.c[3 * v], S.c[3 * v + 1], S.c[3 * v + 2]);
  double k[MAX_INTR];
#pragma unroll
  for (int i = 0; i < MAX_INTR; ++i) k[i] = S.k[i];
  double acc[CC_NACC][2];
#pragma unroll
  for (int i = 0; i < CC_NACC; ++i) { acc[i][0] = 0.0; acc[i][1] = 0.0; }
  double cost = 0.0, esum = 0.0;
  for (int base = c0; base < c1; base += 32) {
    const int c = base + lane;
    const int nact = min(32, c1 - base);
    double rx[CC_COLS], ry[CC_COLS];
    if (JAC) {
#pragma unroll
      for (int i = 0; i < CC_COLS; ++i) { rx[i] = 0.0; ry[i] = 0.0; }
    }
    if (RS && c < c1) {
      const double4 Xb = Q.board[Q.pid[c]];
      const double iw = 1.0 / Xb.w;
      const double* vel = rs.vel + 6 * v;
      RsMotion m; m.w = v3(vel[0], vel[1], vel[2]); m.u = v3(vel[3], vel[4], vel[5]);
      const double2 uv = Q.uv[c];
      double r0, r1, J0[6], J1[6], Jk0[MAX_INTR], Jk1[MAX_INTR];
      const bool ok = rs_camera_residual(Q.model, k, q, cc, v3(Xb.x * iw, Xb.y * iw, Xb.z * iw), m, uv.y * rs.line_delay, uv, r0, r1,
                                         JAC ? J0 : nullptr, JAC ? J1 : nullptr, JAC ? Jk0 : nullptr, JAC ? Jk1 : nullptr);
      if (!ok) { cost += 1e10; esum += 1e10; }
      else {
        const double s = r0 * r0 + r1 * r1, rn = sqrt(s);
        const bool in = rn <= Q.huber;
        cost += in ? 0.5 * s : Q.huber * rn - 0.5 * Q.huber * Q.huber;
        esum += rn;
        if (JAC) {
          const double sw = in ? 1.0 : sqrt(Q.huber / rn);
          if (Q.pose_free)
#pragma unroll
            for (int i = 0; i < 6; ++i) { rx[i] = sw * J0[i]; ry[i] = sw * J1[i]; }
#pragma unroll
          for (int i = 0; i < MAX_INTR; ++i) if ((Q.intr_mask >> i) & 1u) { rx[6 + i] = sw * Jk0[i]; ry[6 + i] = sw * Jk1[i]; }
          rx[CC_RES] = sw * r0; ry[CC_RES] = sw * r1;
        }
      }
    } else if (!RS && c < c1) {
      const double4 Xb = Q.board[Q.pid[c]];
      const double iw = 1.0 / Xb.w;
      const V3 d = v3(Xb.x * iw, Xb.y * iw, Xb.z * iw) - cc;
      const V3 pc = qrot(q, d);
      ProjK pkk;
      Proj pr;
      if (JAC) pr = project_with_k(Q.model, k, pc, true, &pkk); else pr = project(Q.model, k, pc, true);
      if (!pr.ok) { cost += 1e10; esum += 1e10; }   // outside the model's domain: theia's residual functor fails, the step is refused
      else {
        const double r0 = pr.u - Q.uv[c].x, r1 = pr.v - Q.uv[c].y, s = r0 * r0 + r1 * r1, rn = sqrt(s);
        // ceres::HuberLoss(a): rho(s) = s (s <= a^2), 2 a sqrt(s) - a^2 beyond; cost = rho / 2; rho'' <= 0, so the corrector only
        // rescales residual and Jacobian by sqrt(rho')
        const bool in = rn <= Q.huber;
        cost += in ? 0.5 * s : Q.huber * rn - 0.5 * Q.huber * Q.huber;
        esum += rn;
        if (JAC) {
          const double sw = in ? 1.0 : sqrt(Q.huber / rn);
          const V3 a0 = v3(pr.J[0], pr.J[1], pr.J[2]), a1 = v3(pr.J[3], pr.J[4], pr.J[5]);
          if (Q.pose_free) {
            // pc = R exp(delta) (X - c):  d pc / d delta = -R [d]x,  d pc / d c = -R   =>  rows  d x (R^T a)  and  -(R^T a)
            const V3 t0 = qrot_inv(q, a0), t1 = qrot_inv(q, a1);
            const V3 b0 = cross(d, t0), b1 = cross(d, t1);
            rx[0] = sw * b0.x; rx[1] = sw * b0.y; rx[2] = sw * b0.z; rx[3] = -sw * t0.x; rx[4] = -sw * t0.y; rx[5] = -sw * t0.z;
            ry[0] = sw * b1.x; ry[1] = sw * b1.y; ry[2] = sw * b1.z; ry[3] = -sw * t1.x; ry[4] = -sw * t1.y; ry[5] = -sw * t1.z;
          }
#pragma unroll
          for (int i = 0; i < MAX_INTR; ++i) if ((Q.intr_mask >> i) & 1u) { rx[6 + i] = sw * pkk.Jk[jk_at(0, i)]; ry[6 + i] = sw * pkk.Jk[jk_at(1, i)]; }
          rx[CC_RES] = sw * r0; ry[CC_RES] = sw * r1;
        }
      }
    }
    if (JAC) {
      const int nsteps = (nact + 3) >> 2;
#pragma unroll
      for (int i = 0; i < CC_COLS; ++i) tile[i * LDT + lane] = rx[i];
      __syncwarp();
      syrk_tile(tile, nsteps, acc);
      __syncwarp();
#pragma unroll
      for (int i = 0; i < CC_COLS; ++i) tile[i * LDT + lane] = ry[i];
      __syncwarp();
      syrk_tile(tile, nsteps, acc);
      __syncwarp();
    }
  }
  cost = warp_sum(cost); esum = warp_sum(esum);
  if (JAC) {
    // fragment (bi, bj) of lane l holds entries (I, J), (I, J + 1) with I = 8 bi + l / 4, J = 8 bj + 2 (l % 4): keep the upper triangle
    int idx = 0;
#pragma unroll
    for (int bi = 0; bi < CC_NB; ++bi)
#pragma unroll
      for (int bj = bi; bj < CC_NB; ++bj) {
        const int I = 8 * bi + (lane >> 2);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int J = 8 * bj + 2 * (lane & 3) + e;
          if (I <= J && J < CC_COLS) {
            const int o = pk(I, J);
            blocks[(size_t)slot * CC_PACK + o] = acc[idx][e];
            if (I >= 6 && acc[idx][e] != 0.0) atomicAdd(&sys[o], acc[idx][e]);
          }
        }
        ++idx;
      }
    if (lane == 0) atomicAdd(&sys[CC_PACK], cost);
  } else if (lane == 0) {
    atomicAdd(cost_out, cost);
    if (view_err) view_err[v] = c1 > c0 ? esum / (double)(c1 - c0) : 0.0;
  }
}

// effective (unscaled) LM damping of a column with Jacobi scaling s:  clamp(s^2 H_ii, min, max) / radius / s^2   (Ceres'
// LevenbergMarquardtStrategy applied to the column-scaled Jacobian)
ICC_D double lm_damping(double hii, double s, double radius, double mind, double maxd) {
  return fmin(fmax(s * s * hii, mind), maxd) / (radius * s * s);
}

constexpr int RED_THREADS = 64;
__global__ void __launch_bounds__(RED_THREADS) camcal_reduce_kernel(CamCalProblem Q, const double* __restrict__ blocks, double* __restrict__ red, double* __restrict__ Y,
                                                           double* __restrict__ scale, int compute_scale, double radius, double mind, double maxd, double* __restrict__ scal) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  const bool live = slot < Q.n_active && Q.pose_free;
  double Yl[MAX_INTR + 1][6];   // Yl[c] = column c of Y = A^-1 [H_pk | g_p]: one right-hand side of the 6x6 system each
  double Hpk[6][MAX_INTR];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int c = 0; c <= MAX_INTR; ++c) Yl[c][i] = 0.0;
#pragma unroll
    for (int c = 0; c < MAX_INTR; ++c) Hpk[i][c] = 0.0;
  }
  double gmax = 0.0;
  if (live) {
    const double* B = blocks + (size_t)slot * CC_PACK;
    double A[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
      for (int j = 0; j < 6; ++j) if (j >= i) { A[j][i] = B[pk(i, j)]; }
#pragma unroll
      for (int c = 0; c < MAX_INTR; ++c) { Hpk[i][c] = B[pk(i, 6 + c)]; Yl[c][i] = Hpk[i][c]; }
      Yl[MAX_INTR][i] = B[pk(i, CC_RES)];
      gmax = fmax(gmax, fabs(Yl[MAX_INTR][i]));
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double s = compute_scale ? 1.0 / (1.0 + sqrt(A[i][i])) : scale[6 * slot + i];
      if (compute_scale) scale[6 * slot + i] = s;
      A[i][i] += lm_damping(A[i][i], s, radius, mind, maxd);
    }
    const bool ok = chol_factor<6>(A);
#pragma unroll
    for (int c = 0; c <= MAX_INTR; ++c) chol_substitute<6>(A, Yl[c]);
    if (!ok) atomicAdd(&scal[CC_FAIL], 1.0);
    double* Yo = Y + (size_t)slot * CC_Y;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int c = 0; c <= MAX_INTR; ++c) Yo[i * (MAX_INTR + 1) + c] = Yl[c][i];
  } else if (slot < Q.n_active) {
    double* Yo = Y + (size_t)slot * CC_Y;
    for (int i = 0; i < CC_Y; ++i) Yo[i] = 0.0;
  }
  // Schur complement of this view onto the intrinsics: -H_pk^T Y  (matrix and gradient part); the CC_RED sums of the CTA's views are
  // formed through shared memory (one column per thread, then one thread per output), RED_ROWS of them per pass, one RED.ADD.F64 each
  constexpr int RED_ROWS = 65;
  __shared__ double part[RED_ROWS][RED_THREADS + 1];
  for (int o0 = 0; o0 < CC_RED; o0 += RED_ROWS) {
    int o = 0;
#pragma unroll
    for (int a = 0; a < MAX_INTR; ++a) {
#pragma unroll
      for (int b = 0; b <= MAX_INTR; ++b) if (b >= a) {
        if (o >= o0 && o < o0 + RED_ROWS) {
          double sacc = 0.0;
#pragma unroll
          for (int i = 0; i < 6; ++i) sacc -= Hpk[i][a] * Yl[b][i];
          part[o - o0][threadIdx.x] = sacc;
        }
        ++o;
      }
    }
    __syncthreads();
    for (int o = o0 + threadIdx.x; o < o0 + RED_ROWS && o < CC_RED; o += RED_THREADS) {
      double sacc = 0.0;
      for (int t = 0; t < RED_THREADS; ++t) sacc += part[o - o0][t];
      // o enumerates (a, b >= a) row by row with b = MAX_INTR the gradient column
      int a = 0, r = o; while (r >= MAX_INTR + 1 - a) { r -= MAX_INTR + 1 - a; ++a; }
      const int b = a + r;
      if (sacc != 0.0) atomicAdd(&red[b < MAX_INTR ? pkr(a, b) : CC_RED_G + a], sacc);
    }
    __syncthreads();
  }
  gmax = warp_max(gmax);
  if (lane == 0 && gmax > 0.0) atomic_max_nonneg(&scal[CC_GRAD_MAX], gmax);
}

__global__ void camcal_solve_kernel(CamCalProblem Q, CamCalState cur, CamCalState cand, const double* __restrict__ sys, const double* __restrict__ red,
                                    double* __restrict__ scale_k, int compute_scale, double radius, double mind, double maxd, double* __restrict__ dk, double* __restrict__ scal) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double A[MAX_INTR][MAX_INTR], b[MAX_INTR], D[MAX_INTR], g[MAX_INTR];
  double gmax = 0.0;
  for (int a = 0; a < MAX_INTR; ++a) {
    const bool act = (Q.intr_mask >> a) & 1u;
    g[a] = act ? sys[pk(6 + a, CC_RES)] : 0.0;
    gmax = fmax(gmax, fabs(g[a]));
    for (int c = a; c < MAX_INTR; ++c) { const double v = sys[pk(6 + a, 6 + c)] + red[pkr(a, c)]; A[c][a] = v; A[a][c] = v; }
    if (act) {
      const double hii = sys[pk(6 + a, 6 + a)];
      const double s = compute_scale ? 1.0 / (1.0 + sqrt(hii)) : scale_k[a];
      if (compute_scale) scale_k[a] = s;
      D[a] = lm_damping(hii, s, radius, mind, maxd);
      A[a][a] += D[a];
      b[a] = -(g[a] + red[CC_RED_G + a]);
    } else { D[a] = 0.0; b[a] = 0.0; }
  }
  for (int a = 0; a < MAX_INTR; ++a) if (!((Q.intr_mask >> a) & 1u)) { for (int c = 0; c < MAX_INTR; ++c) { A[a][c] = 0.0; A[c][a] = 0.0; } A[a][a] = 1.0; }
  const bool ok = chol_solve<MAX_INTR>(A, b);
  double gd = 0.0, dd = 0.0, st = 0.0, xs = 0.0;
  for (int a = 0; a < MAX_INTR; ++a) {
    dk[a] = b[a]; cand.k[a] = cur.k[a] + b[a];
    gd += g[a] * b[a]; dd += D[a] * b[a] * b[a]; st += b[a] * b[a]; xs += cur.k[a] * cur.k[a];
  }
  if (!ok) atomicAdd(&scal[CC_FAIL], 1.0);
  atomicAdd(&scal[CC_G_DELTA], gd); atomicAdd(&scal[CC_D_DELTA], dd); atomicAdd(&scal[CC_STEP_SQ], st); atomicAdd(&scal[CC_X_SQ], xs);
  if (gmax > 0.0) atomic_max_nonneg(&scal[CC_GRAD_MAX], gmax);
  scal[CC_X_COST] = sys[CC_PACK];
}

__global__ void __launch_bounds__(128) camcal_update_kernel(CamCalProblem Q, CamCalState cur, CamCalState cand, const double* __restrict__ blocks, const double* __restrict__ Y,
                                                           const double* __restrict__ dk, const double* __restrict__ scale, double radius, double mind, double maxd, double* __restrict__ scal) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  double gd = 0.0, dd = 0.0, st = 0.0, xs = 0.0;
  if (slot < Q.n_active) {
    const int v = Q.active[slot];
    const Q4 q = q4(cur.q[4 * v], cur.q[4 * v + 1], cur.q[4 * v + 2], cur.q[4 * v + 3]);
    const V3 c = v3(cur.c[3 * v], cur.c[3 * v + 1], cur.c[3 * v + 2]);
    double dp[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (Q.pose_free) {
      const double* Yi = Y + (size_t)slot * CC_Y;
      const double* B = blocks + (size_t)slot * CC_PACK;
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        double s = Yi[i * (MAX_INTR + 1) + MAX_INTR];
#pragma unroll
        for (int a = 0; a < MAX_INTR; ++a) s += Yi[i * (MAX_INTR + 1) + a] * dk[a];
        dp[i] = -s;
        const double hii = B[pk(i, i)];
        gd += B[pk(i, CC_RES)] * dp[i];
        dd += lm_damping(hii, scale[6 * slot + i], radius, mind, maxd) * dp[i] * dp[i];
        st += dp[i] * dp[i];
      }
    }
    const Q4 qn = qnormalized(qmul(q, so3_exp(v3(dp[0], dp[1], dp[2]))));
    cand.q[4 * v] = qn.x; cand.q[4 * v + 1] = qn.y; cand.q[4 * v + 2] = qn.z; cand.q[4 * v + 3] = qn.w;
    cand.c[3 * v] = c.x + dp[3]; cand.c[3 * v + 1] = c.y + dp[4]; cand.c[3 * v + 2] = c.z + dp[5];
    xs = 1.0 + dot(c, c);
  }
  gd = warp_sum(gd); dd = warp_sum(dd); st = warp_sum(st); xs = warp_sum(xs);
  if (lane == 0) { atomicAdd(&scal[CC_G_DELTA], gd); atomicAdd(&scal[CC_D_DELTA], dd); atomicAdd(&scal[CC_STEP_SQ], st); atomicAdd(&scal[CC_X_SQ], xs); }
}

// theia::CameraIntrinsicsModel::GetSubsetFromOptimizeIntrinsicsType per model, as bit masks over Theia's parameter order
struct IntrinsicSubsets { unsigned focal, aspect, principal, radial, tangential; };
IntrinsicSubsets intrinsic_subsets(int model) {
  auto bits = [](std::initializer_list<int> l) { unsigned m = 0; for (int i : l) m |= 1u << i; return m; };
  switch (model) {
    case CAM_PINHOLE: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6}), 0u};
    case CAM_PINHOLE_RADTAN: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7}), bits({8, 9})};
    case CAM_FISHEYE: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7, 8}), 0u};
    case CAM_FOV: return {bits({0}), bits({1}), bits({2, 3}), bits({4}), 0u};
    case CAM_DIVISION_UNDISTORTION: return {bits({0}), bits({1}), bits({2, 3}), bits({4}), 0u};
    case CAM_DOUBLE_SPHERE: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6}), 0u};
    case CAM_EXTENDED_UNIFIED: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6}), 0u};
    case CAM_OMNI_RADTAN: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7}), bits({8, 9})};   // radial = xi, k1, k2
    case CAM_SCARAMUZZA: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7}), bits({2, 8})};    // radial = a2, a3, a4; the stretch e, d as tangential
    case CAM_PINHOLE_RATIONAL: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7, 10, 11, 12}), bits({8, 9})};   // radial = k1..k6
    case CAM_FISHEYE_RADTAN: return {bits({0}), bits({1}), bits({3, 4}), bits({5, 6, 7, 8, 9, 10}), bits({11, 12})};      // radial = k1..k6
    default: return {0u, 0u, 0u, 0u, 0u};
  }
}

}  // namespace

// with_jacobian: per-view packed blocks (n_active x CC_PACK) + the intrinsics part and the cost summed into sys[CC_PACK + 1];
// otherwise cost only into *cost_out and (optional) the per-view mean reprojection error [px] into view_err (indexed by view)
// rs.vel == nullptr: the global shutter
void launch_camcal_accumulate(const CamCalProblem& Q, const CamCalState& S, bool with_jacobian, double* blocks, double* sys, double* cost_out, double* view_err, const CamCalRs& rs,
                              cudaStream_t st) {
  if (Q.n_active <= 0) return;
  const int grid = (Q.n_active + 3) / 4;
  if (rs.vel) {
    if (with_jacobian) camcal_accumulate_kernel<true, true><<<grid, 128, 0, st>>>(Q, S, blocks, sys, nullptr, nullptr, rs);
    else camcal_accumulate_kernel<false, true><<<grid, 128, 0, st>>>(Q, S, nullptr, nullptr, cost_out, view_err, rs);
  } else {
    if (with_jacobian) camcal_accumulate_kernel<true, false><<<grid, 128, 0, st>>>(Q, S, blocks, sys, nullptr, nullptr, CamCalRs{});
    else camcal_accumulate_kernel<false, false><<<grid, 128, 0, st>>>(Q, S, nullptr, nullptr, cost_out, view_err, CamCalRs{});
  }
  count_launch();
}

// one damped step: per-view Schur elimination, reduced intrinsics system, back-substitution into the candidate state
void launch_camcal_step(const CamCalProblem& Q, const CamCalState& cur, const CamCalState& cand, const double* blocks, const double* sys, double* red /* CC_RED */, double* Y,
                        double* scale /* 6 n_active + MAX_INTR */, int compute_scale, double radius, double min_diag, double max_diag, double* dk /* MAX_INTR */, double* scal, cudaStream_t st) {
  if (Q.n_active <= 0) return;
  const int grid = (Q.n_active + 127) / 128;
  camcal_reduce_kernel<<<(Q.n_active + RED_THREADS - 1) / RED_THREADS, RED_THREADS, 0, st>>>(Q, blocks, red, Y, scale, compute_scale, radius, min_diag, max_diag, scal);
  count_launch();
  camcal_solve_kernel<<<1, 32, 0, st>>>(Q, cur, cand, sys, red, scale + 6 * (size_t)Q.n_active, compute_scale, radius, min_diag, max_diag, dk, scal);
  count_launch();
  camcal_update_kernel<<<grid, 128, 0, st>>>(Q, cur, cand, blocks, Y, dk, scale, radius, min_diag, max_diag, scal);
  count_launch();
}

// ---- host driver of row f4 (icc_calibrate_camera): CameraCalibrator, src/core/camera_calibrator.cc ------------------------------
#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status calibrate_camera(cudaStream_t st, int model, int W, int H, int np, const double* points, int nv, const int32_t* off, const int32_t* ids, const double* uv,
                            const double* q_init, const double* p_init, const int32_t* init_valid, double focal_init, double distortion_init, const icc_camcal_options* options,
                            double* intr_out, double* q_out, double* p_out, double* err_out, int32_t* used_out, icc_camcal_summary& S, std::vector<double>& points_out, std::string& err,
                            const CamCalShutter& shutter) {
  using clk = std::chrono::steady_clock;
  const auto t_start = clk::now();
  memset(&S, 0, sizeof S);
  const int launches0 = kernel_launch_count();
  // ---- inputs to the device ------------------------------------------------------------------------------------------------
  BoardViews B;
  icc_status rc = upload_board_views(st, np, points, nv, off, ids, uv, B, err); if (rc != ICC_OK) return rc;
  const int nc = B.nc;
  icc_camcal_options o; memset(&o, 0, sizeof o); if (options) o = *options;
  if (o.grid_size < 0.0) o.grid_size = 0.04;
  if (o.min_num_views <= 0) o.min_num_views = 10;
  if (o.max_num_iterations <= 0) o.max_num_iterations = 100;
  if (!(o.function_tolerance > 0.0)) o.function_tolerance = 1e-6;
  if (!(o.parameter_tolerance > 0.0)) o.parameter_tolerance = 1e-8;
  if (!(o.gradient_tolerance > 0.0)) o.gradient_tolerance = 1e-10;
  if (!(o.huber_width > 0.0)) o.huber_width = 1.345;
  if (!(o.max_view_error_stage1_px > 0.0)) o.max_view_error_stage1_px = 5.0;
  if (!(o.max_view_error_final_px > 0.0)) o.max_view_error_final_px = 2.0;
  DevBuf<int> d_active; CU(d_active.alloc(nv));
  // rolling shutter: the views' fixed velocities on the device; every bundle adjustment (the initialiser's included) and the board points see
  // each corner at its row time
  DevBuf<double> d_vel;
  const bool rolling = shutter.line_delay > 0.0;
  if (rolling) { CU(d_vel.alloc(6 * (size_t)nv)); CU(cudaMemcpyAsync(d_vel.p, shutter.vel, 6 * (size_t)nv * sizeof(double), cudaMemcpyHostToDevice, st)); }
  const CamCalRs rs{rolling ? d_vel.p : nullptr, rolling ? shutter.line_delay : 0.0};
  const double cx0 = W / 2.0, cy0 = H / 2.0;                       // AddView (:99)
  // ---- initial focal length and poses ----------------------------------------------------------------------------------------
  std::vector<double> q0(4 * (size_t)nv), p0(3 * (size_t)nv); std::vector<int> ok0(nv, 1);
  const bool need_focal = !(focal_init > 0.0), need_poses = !q_init || !p_init;
  double f0 = focal_init;
  if (need_focal || need_poses) {
    PoseProblem PQ; memset(&PQ, 0, sizeof PQ);
    PQ.model = CAM_PINHOLE; PQ.n_frames = nv; PQ.n_points = np; PQ.min_points = 6;
    PQ.board = B.board.p; PQ.f_off = B.off.p; PQ.pid = B.pid.p; PQ.thresh_sq = 1e300; PQ.max_err = 1e300;   // every corner takes part
    PQ.lm_rel_tol = 1e-6;                                                                                  // these poses only start the bundle adjustment
    if (need_focal) {
      DevBuf<double> d_f2; CU(d_f2.alloc(nv));
      launch_board_focal(PQ, B.uv.p, cx0, cy0, B.xy.p, B.use.p, d_f2.p, st);
      std::vector<double> f2(nv);
      CU(cudaMemcpyAsync(f2.data(), d_f2.p, (size_t)nv * sizeof(double), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      std::vector<double> fs; for (double v : f2) if (v > 0.0 && std::isfinite(v)) fs.push_back(std::sqrt(v));
      if (fs.empty()) { err = "no view yields a focal length estimate (fronto-parallel or degenerate views only)"; return ICC_ERR_NUMERIC; }
      f0 = median_like_reference(fs);
    }
    if (need_poses) {
      launch_pinhole_normalize(nc, B.uv.p, cx0, cy0, f0, B.xy.p, B.ok.p, st);
      launch_board_poses(PQ, B.xy.p, B.ok.p, B.use.p, B.q.p, B.p.p, B.e.p, B.valid.p, st);
      rc = read_poses(st, B, q0.data(), p0.data(), nullptr, ok0.data(), err); if (rc != ICC_OK) return rc;
    }
  }
  if (!need_poses) {
    memcpy(q0.data(), q_init, 4 * (size_t)nv * sizeof(double)); memcpy(p0.data(), p_init, 3 * (size_t)nv * sizeof(double));
    if (init_valid) for (int i = 0; i < nv; ++i) ok0[i] = init_valid[i] != 0;
  }
  // ---- state: R_cw = conj(q_wc), camera centre, shared intrinsics ---------------------------------------------------------------
  std::vector<double> qs(4 * (size_t)nv), k0(MAX_INTR, 0.0);
  for (int v = 0; v < nv; ++v) {
    const Q4 q = qnormalized(q4(q0[4 * v], q0[4 * v + 1], q0[4 * v + 2], q0[4 * v + 3]));
    qs[4 * v] = -q.x; qs[4 * v + 1] = -q.y; qs[4 * v + 2] = -q.z; qs[4 * v + 3] = q.w;
  }
  // the internal initialiser refines (focal length, division distortion, poses) jointly before the target model takes over -- the
  // role of utils::initialize_radial_undistortion_camera (:283-306), which hands the reference a focal length and a division-model
  // distortion for every non-pinhole model
  const bool prestage = need_poses && need_focal && model != CAM_PINHOLE && model != CAM_PINHOLE_RADTAN;
  std::vector<int> active;
  for (int v = 0; v < nv; ++v) if (ok0[v]) active.push_back(v);
  S.n_views_initialized = (int)active.size();
  if (prestage) { k0[0] = f0; k0[1] = 1.0; k0[2] = cx0; k0[3] = cy0; k0[4] = -1e-2 / ((double)W * W + (double)H * H); }
  DevBuf<double> d_q[2], d_c[2], d_k[2], d_blocks, d_Y, d_scale, d_sys, d_red, d_dk, d_scal, d_verr;
  for (int i = 0; i < 2; ++i) { CU(d_q[i].upload(qs)); CU(d_c[i].upload(p0)); CU(d_k[i].upload(k0)); }
  const size_t na0 = std::max<size_t>(1, active.size());
  CU(d_blocks.alloc(na0 * CC_PACK)); CU(d_Y.alloc(na0 * CC_Y)); CU(d_scale.alloc(6 * na0 + MAX_INTR)); CU(d_sys.alloc(CC_PACK + 1)); CU(d_red.alloc(CC_RED));
  CU(d_dk.alloc(MAX_INTR)); CU(d_scal.alloc(CC_SCAL_COUNT)); CU(d_verr.alloc(nv));
  int cur = 0;
  CamCalProblem Q; memset(&Q, 0, sizeof Q);
  Q.model = model; Q.n_points = np; Q.huber = o.huber_width; Q.board = B.board.p; Q.f_off = B.off.p; Q.pid = B.pid.p; Q.uv = B.uv.p; Q.active = d_active.p;
  auto state = [&](int i) { CamCalState s; s.q = d_q[i].p; s.c = d_c[i].p; s.k = d_k[i].p; return s; };
  auto set_active = [&]() -> icc_status {
    Q.n_active = (int)active.size();
    if (!active.empty()) CU(cudaMemcpyAsync(d_active.p, active.data(), active.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));   // `active` may be modified by the caller right after
    return ICC_OK;
  };
  std::vector<double> verr(nv, 0.0);
  // GetReprojErrorOfView for every active view at the current state
  auto view_errors = [&]() -> icc_status {
    CU(cudaMemsetAsync(d_scal.p, 0, CC_SCAL_COUNT * sizeof(double), st));
    launch_camcal_accumulate(Q, state(cur), false, nullptr, nullptr, d_scal.p + CC_CAND_COST, d_verr.p, rs, st);
    CU(cudaMemcpyAsync(verr.data(), d_verr.p, (size_t)nv * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return ICC_OK;
  };
  // RemoveViewsReprojError (:59-76)
  auto remove_views = [&](double max_err) -> icc_status {
    icc_status r = view_errors(); if (r != ICC_OK) return r;
    std::vector<int> keep; for (int v : active) if (!(verr[v] > max_err)) keep.push_back(v);
    active.swap(keep);
    return set_active();
  };
  // theia::BundleAdjustViews: Levenberg-Marquardt with Ceres' trust-region logic; one device->host read-back per iteration
  auto bundle_adjust = [&](unsigned mask, bool pose_free, int stage) -> icc_status {
    Q.intr_mask = mask; Q.pose_free = pose_free ? 1 : 0;
    if (Q.n_active == 0 || (mask == 0u && !pose_free)) { if (stage >= 0) S.termination[stage] = 3; return ICC_OK; }
    TrOptions to = ceres_default_options();   // theia::BundleAdjustmentOptions: the Ceres defaults but for these
    to.function_tolerance = o.function_tolerance; to.parameter_tolerance = o.parameter_tolerance; to.gradient_tolerance = o.gradient_tolerance;
    to.max_iterations = o.max_num_iterations;
    TrustRegion T = tr_start(to);
    double sc[CC_SCAL_COUNT];
    while (tr_continue(T)) {
      const bool fresh = T.jacobian_stale != 0;
      if (fresh) {
        CU(cudaMemsetAsync(d_sys.p, 0, (CC_PACK + 1) * sizeof(double), st));
        launch_camcal_accumulate(Q, state(cur), true, d_blocks.p, d_sys.p, nullptr, nullptr, rs, st);
      }
      CU(cudaMemsetAsync(d_red.p, 0, CC_RED * sizeof(double), st));
      CU(cudaMemsetAsync(d_scal.p, 0, CC_SCAL_COUNT * sizeof(double), st));
      launch_camcal_step(Q, state(cur), state(1 - cur), d_blocks.p, d_sys.p, d_red.p, d_Y.p, d_scale.p, T.iterations == 0 ? 1 : 0, T.radius, to.min_diagonal, to.max_diagonal, d_dk.p, d_scal.p, st);
      launch_camcal_accumulate(Q, state(1 - cur), false, nullptr, nullptr, d_scal.p + CC_CAND_COST, nullptr, rs, st);
      CU(cudaMemcpyAsync(sc, d_scal.p, sizeof sc, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      if (fresh) {
        if (T.iterations == 0 && !std::isfinite(sc[CC_X_COST])) { err = "non-finite initial cost"; return ICC_ERR_NUMERIC; }
        if (!tr_jacobian(T, sc[CC_X_COST], sc[CC_GRAD_MAX])) break;
      }
      if (tr_step(T, sc[CC_FAIL] == 0.0, 0.5 * (sc[CC_D_DELTA] - sc[CC_G_DELTA]), std::sqrt(sc[CC_STEP_SQ]), std::sqrt(sc[CC_X_SQ])) && tr_candidate(T, sc[CC_CAND_COST]))
        cur = 1 - cur;
    }
    // both state copies must agree on everything outside the last step (inactive views never move; the intrinsics / poses of
    // a rejected candidate are stale): bring the spare copy back to the current state
    CU(cudaMemcpyAsync(d_q[1 - cur].p, d_q[cur].p, 4 * (size_t)nv * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(d_c[1 - cur].p, d_c[cur].p, 3 * (size_t)nv * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(d_k[1 - cur].p, d_k[cur].p, MAX_INTR * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (stage == 0) S.initial_cost = T.initial_cost;
    if (stage >= 0) { S.final_cost[stage] = T.cost; S.iterations[stage] = T.iterations; S.termination[stage] = T.termination; } else S.init_iterations = T.iterations;
    return ICC_OK;
  };
  auto finish = [&](bool success) -> icc_status {
    icc_status r = view_errors(); if (r != ICC_OK) return r;
    std::vector<double> qh(4 * (size_t)nv), ch(3 * (size_t)nv), kh(MAX_INTR);
    CU(cudaMemcpy(qh.data(), d_q[cur].p, qh.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(ch.data(), d_c[cur].p, ch.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(kh.data(), d_k[cur].p, MAX_INTR * sizeof(double), cudaMemcpyDeviceToHost));
    for (int v = 0; v < nv; ++v) {
      q_out[4 * v] = -qh[4 * v]; q_out[4 * v + 1] = -qh[4 * v + 1]; q_out[4 * v + 2] = -qh[4 * v + 2]; q_out[4 * v + 3] = qh[4 * v + 3];
      for (int d = 0; d < 3; ++d) p_out[3 * v + d] = ch[3 * v + d];
      used_out[v] = 0; if (err_out) err_out[v] = 0.0;
    }
    double tot = 0.0;
    for (int v : active) { used_out[v] = 1; if (err_out) err_out[v] = verr[v]; tot += verr[v]; }
    for (int i = 0; i < std::max(10, camera_num_params(model)); ++i) intr_out[i] = kh[i];   // icc_b200.h: max(10, parameter count) entries
    S.success = success ? 1 : 0; S.n_views_used = (int)active.size();
    S.final_reproj_error = active.empty() ? 0.0 : tot / (double)active.size();                 // :352-366
    S.gpu_launches = kernel_launch_count() - launches0;
    S.seconds_total = std::chrono::duration<double>(clk::now() - t_start).count();
    return ICC_OK;
  };
  rc = set_active(); if (rc != ICC_OK) return rc;
  if (prestage) {
    Q.model = CAM_DIVISION_UNDISTORTION;
    rc = bundle_adjust((1u << 0) | (1u << 4), true, -1); if (rc != ICC_OK) return rc;
    Q.model = model;
    double kd[MAX_INTR];
    CU(cudaMemcpy(kd, d_k[cur].p, sizeof kd, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(p0.data(), d_c[cur].p, p0.size() * sizeof(double), cudaMemcpyDeviceToHost));
    if (kd[0] > 0.0 && std::isfinite(kd[0])) { f0 = kd[0]; if (model == CAM_DIVISION_UNDISTORTION) distortion_init = kd[4]; }
  }
  S.focal_length_init = f0;
  // ---- grid filter in file order (:313-325): a view is taken iff no accepted camera position lies within grid_size ---------------
  // (the reference scans all accepted positions; a hash grid with cells of grid_size visits only the 27 cells that can hold one
  // -- same decisions, linear time)
  if (o.grid_size > 0.0) {
    std::vector<int> sel;
    std::unordered_map<uint64_t, std::vector<int>> cells;
    const double inv = 1.0 / o.grid_size;
    bool hashable = true;
    for (int v : active) for (int d = 0; d < 3; ++d) if (!(std::fabs(p0[3 * v + d] * inv) < 1e6)) hashable = false;   // 21 bits per axis
    auto key = [](int64_t x, int64_t y, int64_t z) { return (uint64_t)((x + (1 << 20)) & 0x1fffff) << 42 | (uint64_t)((y + (1 << 20)) & 0x1fffff) << 21 | (uint64_t)((z + (1 << 20)) & 0x1fffff); };
    auto close_to = [&](int v, int a) { const double dx = p0[3 * v] - p0[3 * a], dy = p0[3 * v + 1] - p0[3 * a + 1], dz = p0[3 * v + 2] - p0[3 * a + 2]; return std::sqrt(dx * dx + dy * dy + dz * dz) < o.grid_size; };
    for (int v : active) {
      bool take = true;
      if (hashable) {
        const int64_t cx = (int64_t)std::floor(p0[3 * v] * inv), cy = (int64_t)std::floor(p0[3 * v + 1] * inv), cz = (int64_t)std::floor(p0[3 * v + 2] * inv);
        for (int64_t x = cx - 1; x <= cx + 1 && take; ++x) for (int64_t y = cy - 1; y <= cy + 1 && take; ++y) for (int64_t z = cz - 1; z <= cz + 1 && take; ++z) {
          auto it = cells.find(key(x, y, z));
          if (it != cells.end()) for (int a : it->second) if (close_to(v, a)) { take = false; break; }
        }
        if (take) cells[key(cx, cy, cz)].push_back(v);
      } else {
        for (int a : sel) if (close_to(v, a)) { take = false; break; }
      }
      if (take) sel.push_back(v);
    }
    active.swap(sel);
  }
  S.n_views_selected = (int)active.size();
  rc = set_active(); if (rc != ICC_OK) return rc;
  // ---- initial intrinsics of the target model (AddView :84-129) --------------------------------------------------------------------
  std::fill(k0.begin(), k0.end(), 0.0);
  k0[0] = f0; k0[1] = 1.0;
  switch (model) {
    case CAM_FOV: case CAM_DIVISION_UNDISTORTION: k0[2] = cx0; k0[3] = cy0; break;
    default: k0[3] = cx0; k0[4] = cy0; break;
  }
  if (model == CAM_DIVISION_UNDISTORTION) k0[4] = distortion_init;
  if (model == CAM_FOV) k0[4] = distortion_init != 0.0 ? distortion_init : 1e-3;   // theia's FOV model has no gradient at omega = 0
  if (model == CAM_DOUBLE_SPHERE) { k0[5] = -0.25; k0[6] = 0.5; }
  if (model == CAM_EXTENDED_UNIFIED) { k0[5] = 0.5; k0[6] = 1.0; }
  if (model == CAM_OMNI_RADTAN) { k0[5] = 1.0; k0[0] = 2.0 * f0; }   // xi = 1, f = (1 + xi) f0: magnification f / (1 + xi) = f0 at the image centre
  if (model == CAM_SCARAMUZZA) k0[5] = -0.25 / f0;                    // the stereographic member a2 = -1 / (4 a0): magnification a0 = f0 at the image centre
  for (int i = 0; i < 2; ++i) CU(cudaMemcpy(d_k[i].p, k0.data(), MAX_INTR * sizeof(double), cudaMemcpyHostToDevice));
  if ((int)active.size() < o.min_num_views) return finish(false);                               // :132-135
  const IntrinsicSubsets sub = intrinsic_subsets(model);
  // 1. focal length and radial distortion, principal point fixed (:146-160)
  rc = bundle_adjust(sub.focal | (model != CAM_PINHOLE ? sub.radial : 0u), true, 0); if (rc != ICC_OK) return rc;
  rc = remove_views(o.max_view_error_stage1_px); if (rc != ICC_OK) return rc;                    // :162
  // 2. principal point, everything else fixed (:164-174)
  rc = bundle_adjust(sub.principal, false, 1); if (rc != ICC_OK) return rc;
  if ((int)active.size() < o.min_num_views) return finish(false);                               // :176-179
  // 3. full optimisation (:181-198)
  const unsigned stage3_mask = sub.principal | sub.focal | sub.aspect | (model == CAM_PINHOLE ? sub.radial : 0u) | (model == CAM_PINHOLE_RADTAN || model == CAM_OMNI_RADTAN || model == CAM_SCARAMUZZA || model == CAM_PINHOLE_RATIONAL ||
                                                                                               model == CAM_FISHEYE_RADTAN ? sub.tangential : 0u);
  rc = bundle_adjust(stage3_mask, true, 2);
  if (rc != ICC_OK) return rc;
  rc = remove_views(o.max_view_error_final_px); if (rc != ICC_OK) return rc;                     // :200
  if ((int)active.size() < o.min_num_views) return finish(false);                                // :202-205
  if (o.optimize_board_points) {                                                                 // :207-216
    // BundleAdjustTracks: every camera constant, one warp per board point over its observations in the remaining views ...
    std::vector<int> obs_view(std::max(1, nc), -1);
    for (int v : active) for (int c = off[v]; c < off[v + 1]; ++c) obs_view[c] = v;
    PointProblem PQ; memset(&PQ, 0, sizeof PQ);
    PQ.model = model; CU(cudaMemcpy(PQ.intr, d_k[cur].p, MAX_INTR * sizeof(double), cudaMemcpyDeviceToHost));
    PQ.normalized = 0; PQ.n_points = np; PQ.min_obs = 1; PQ.huber = o.huber_width;
    PQ.board_in = B.board.p; PQ.meas = B.uv.p; PQ.q_cw = d_q[cur].p; PQ.cam_c = d_c[cur].p;
    const RsPass rsp{B.uv.p, d_vel.p, shutter.line_delay};
    DevBuf<double4> d_board2; rc = refine_board_points(st, PQ, nc, ids, obs_view, d_board2, points_out, S.n_points_optimized, err, nullptr, rolling ? &rsp : nullptr);
    if (rc != ICC_OK) return rc;
    CU(cudaMemcpyAsync(B.board.p, d_board2.p, (size_t)np * sizeof(double4), cudaMemcpyDeviceToDevice, st));
    // ... then BundleAdjustViews once more with the options of stage 3
    const int it3 = S.iterations[2];
    rc = bundle_adjust(stage3_mask, true, 2); if (rc != ICC_OK) return rc;
    S.iterations[2] += it3;
  }
  return finish(true);
}

}  // namespace icc
