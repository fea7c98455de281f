// Camera intrinsic calibration (sm_90a): bundle adjustment of every view pose + ONE shared intrinsic vector (SURVEY.md §8(f) row f4).
//
// Replaces what the reference delegates to theia::BundleAdjustViews (Ceres, DENSE/SPARSE_SCHUR, autodiff, CPU threads) in
//   CameraCalibrator::RunCalibration            src/core/camera_calibrator.cc:131-219   (three stages, Huber 1.345)
//   utils::GetReprojErrorOfView                 src/utils/utils.cc:163-177              (per-view mean reprojection error)
// with the residual of theia::ReprojectionError (external): r = CameraToPixelCoordinates(intr, R_cw (X - c)) - feature.
//
// Mapping to the machine.  The normal equations are an arrow: 6x6 pose blocks on the diagonal, a border of <= 10 intrinsics.
//   camcal_accumulate_kernel : one WARP per view.  Each lane evaluates one corner (projection + closed-form 2x3 and 2x10
//       Jacobians of icc_camera.cuh, Huber weight) and writes its weighted rows [J_pose | J_intr | r] (17 columns, padded to three
//       8-column blocks) into the warp's shared-memory tile -- x rows, then y rows; each half is folded into the symmetric product
//       with FP64 tensor-core MMAs (mma.sync m8n8k4: 6 block products per 4 rows, the accumulator fragments stay in registers for
//       the whole view), so J^T J, J^T r and r^T r come out of one contraction.  The view's 17x17 block goes to HBM, its intrinsics
//       part is summed into the global system with RED.ADD.F64.
//   camcal_reduce_kernel     : one thread per view: damped 6x6 Cholesky, Y = A^-1 [H_pk | g_p], Schur complement of the view
//       onto the intrinsics, summed over the CTA through shared memory and added to the reduced 10x10 system.
//   camcal_solve_kernel      : the reduced system (<= 10 unknowns) by Cholesky, intrinsics step, candidate intrinsics.
//   camcal_update_kernel     : back-substitution of every view's pose step, candidate poses, step / model-decrease sums.
// The host only sequences these launches and applies Ceres' trust-region logic to eight scalars per iteration (icc_api.cu).
#include "icc_camera.cuh"
#include "icc_kernels.h"

#include <cmath>

namespace icc {

void count_launch();

namespace {

ICC_D double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
ICC_HD int pk(int i, int j) { return i * CC_COLS - i * (i - 1) / 2 + (j - i); }   // packed upper triangle of the 17x17 block, i <= j
ICC_HD int pk10(int a, int b) { return a * 10 - a * (a - 1) / 2 + (b - a); }       // packed upper triangle of the 10x10 reduced system

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

template <bool JAC>
__global__ void __launch_bounds__(128) camcal_accumulate_kernel(CamCalProblem Q, CamCalState S, double* __restrict__ blocks, double* __restrict__ sys,
                                                               double* __restrict__ cost_out, double* __restrict__ view_err) {
  __shared__ double tile_all[JAC ? 4 * CC_TCOLS * LDT : 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = blockIdx.x * 4 + warp;
  if (slot >= Q.n_active) return;
  double* tile = tile_all + (JAC ? warp * CC_TCOLS * LDT : 0);
  if (JAC) { for (int i = lane; i < CC_TCOLS * LDT; i += 32) tile[i] = 0.0; __syncwarp(); }   // the padding columns 17..23 stay zero
  const int v = Q.active[slot];
  const int c0 = Q.f_off[v], c1 = Q.f_off[v + 1];
  const Q4 q = q4(S.q[4 * v], S.q[4 * v + 1], S.q[4 * v + 2], S.q[4 * v + 3]);
  const V3 cc = v3(S.c[3 * v], S.c[3 * v + 1], S.c[3 * v + 2]);
  double k[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) k[i] = S.k[i];
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
    if (c < c1) {
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
          for (int i = 0; i < 10; ++i) if ((Q.intr_mask >> i) & 1u) { rx[6 + i] = sw * pkk.Jk[i]; ry[6 + i] = sw * pkk.Jk[10 + i]; }
          rx[16] = sw * r0; ry[16] = sw * r1;
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
  cost = wsum(cost); esum = wsum(esum);
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
  double Yl[6][11];
  double Hpk[6][10];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int c = 0; c < 11; ++c) Yl[i][c] = 0.0;
#pragma unroll
    for (int c = 0; c < 10; ++c) Hpk[i][c] = 0.0;
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
      for (int c = 0; c < 10; ++c) { Hpk[i][c] = B[pk(i, 6 + c)]; Yl[i][c] = Hpk[i][c]; }
      Yl[i][10] = B[pk(i, 16)];
      gmax = fmax(gmax, fabs(Yl[i][10]));
    }
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double s = compute_scale ? 1.0 / (1.0 + sqrt(A[i][i])) : scale[6 * slot + i];
      if (compute_scale) scale[6 * slot + i] = s;
      A[i][i] += lm_damping(A[i][i], s, radius, mind, maxd);
    }
    // in-place Cholesky (lower), then forward / backward substitution of the 11 right-hand sides
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      double dj = A[j][j];
#pragma unroll
      for (int m = 0; m < 6; ++m) if (m < j) dj -= A[j][m] * A[j][m];
      if (!(dj > 0.0)) { ok = false; dj = 1.0; }
      const double l = sqrt(dj), il = 1.0 / l;
      A[j][j] = l;
#pragma unroll
      for (int i = 0; i < 6; ++i) if (i > j) {
        double s = A[i][j];
#pragma unroll
        for (int m = 0; m < 6; ++m) if (m < j) s -= A[i][m] * A[j][m];
        A[i][j] = s * il;
      }
    }
#pragma unroll
    for (int c = 0; c < 11; ++c) {
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        double s = Yl[i][c];
#pragma unroll
        for (int m = 0; m < 6; ++m) if (m < i) s -= A[i][m] * Yl[m][c];
        Yl[i][c] = s / A[i][i];
      }
#pragma unroll
      for (int ii = 0; ii < 6; ++ii) {
        const int i = 5 - ii;
        double s = Yl[i][c];
#pragma unroll
        for (int m = 0; m < 6; ++m) if (m > i) s -= A[m][i] * Yl[m][c];
        Yl[i][c] = s / A[i][i];
      }
    }
    if (!ok) atomicAdd(&scal[CC_FAIL], 1.0);
    double* Yo = Y + (size_t)slot * CC_Y;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int c = 0; c < 11; ++c) Yo[i * 11 + c] = Yl[i][c];
  } else if (slot < Q.n_active) {
    double* Yo = Y + (size_t)slot * CC_Y;
    for (int i = 0; i < CC_Y; ++i) Yo[i] = 0.0;
  }
  // Schur complement of this view onto the intrinsics: -H_pk^T Y  (matrix and gradient part); the 65 sums of the CTA's views are
  // formed through shared memory (one column per thread, then one thread per output), 65 RED.ADD.F64 per CTA
  __shared__ double part[65][RED_THREADS + 1];
  {
    int o = 0;
#pragma unroll
    for (int a = 0; a < 10; ++a) {
#pragma unroll
      for (int b = 0; b < 11; ++b) if (b >= a) {
        double sacc = 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i) sacc -= Hpk[i][a] * Yl[i][b];
        part[o][threadIdx.x] = sacc;
        ++o;
      }
    }
  }
  __syncthreads();
  for (int o = threadIdx.x; o < 65; o += RED_THREADS) {
    double sacc = 0.0;
    for (int t = 0; t < RED_THREADS; ++t) sacc += part[o][t];
    // o enumerates (a, b >= a) row by row with b = 10 the gradient column
    int a = 0, r = o; while (r >= 11 - a) { r -= 11 - a; ++a; }
    const int b = a + r;
    if (sacc != 0.0) atomicAdd(&red[b < 10 ? pk10(a, b) : 55 + a], sacc);
  }
  gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 16)); gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 8));
  gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 4)); gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 2)); gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, 1));
  if (lane == 0 && gmax > 0.0) atomic_max_nonneg(&scal[CC_GRAD_MAX], gmax);
}

__global__ void camcal_solve_kernel(CamCalProblem Q, CamCalState cur, CamCalState cand, const double* __restrict__ sys, const double* __restrict__ red,
                                    double* __restrict__ scale_k, int compute_scale, double radius, double mind, double maxd, double* __restrict__ dk, double* __restrict__ scal) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double A[10][10], b[10], D[10], g[10];
  bool ok = true;
  double gmax = 0.0;
  for (int a = 0; a < 10; ++a) {
    const bool act = (Q.intr_mask >> a) & 1u;
    g[a] = act ? sys[pk(6 + a, 16)] : 0.0;
    gmax = fmax(gmax, fabs(g[a]));
    for (int c = a; c < 10; ++c) { const double v = sys[pk(6 + a, 6 + c)] + red[pk10(a, c)]; A[c][a] = v; A[a][c] = v; }
    if (act) {
      const double hii = sys[pk(6 + a, 6 + a)];
      const double s = compute_scale ? 1.0 / (1.0 + sqrt(hii)) : scale_k[a];
      if (compute_scale) scale_k[a] = s;
      D[a] = lm_damping(hii, s, radius, mind, maxd);
      A[a][a] += D[a];
      b[a] = -(g[a] + red[55 + a]);
    } else { D[a] = 0.0; b[a] = 0.0; }
  }
  for (int a = 0; a < 10; ++a) if (!((Q.intr_mask >> a) & 1u)) { for (int c = 0; c < 10; ++c) { A[a][c] = 0.0; A[c][a] = 0.0; } A[a][a] = 1.0; }
  for (int j = 0; j < 10; ++j) {
    double dj = A[j][j];
    for (int m = 0; m < j; ++m) dj -= A[j][m] * A[j][m];
    if (!(dj > 0.0)) { ok = false; dj = 1.0; }
    const double l = sqrt(dj);
    A[j][j] = l;
    for (int i = j + 1; i < 10; ++i) { double s = A[i][j]; for (int m = 0; m < j; ++m) s -= A[i][m] * A[j][m]; A[i][j] = s / l; }
  }
  for (int i = 0; i < 10; ++i) { double s = b[i]; for (int m = 0; m < i; ++m) s -= A[i][m] * b[m]; b[i] = s / A[i][i]; }
  for (int i = 9; i >= 0; --i) { double s = b[i]; for (int m = i + 1; m < 10; ++m) s -= A[m][i] * b[m]; b[i] = s / A[i][i]; }
  double gd = 0.0, dd = 0.0, st = 0.0, xs = 0.0;
  for (int a = 0; a < 10; ++a) {
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
        double s = Yi[i * 11 + 10];
#pragma unroll
        for (int a = 0; a < 10; ++a) s += Yi[i * 11 + a] * dk[a];
        dp[i] = -s;
        const double hii = B[pk(i, i)];
        gd += B[pk(i, 16)] * dp[i];
        dd += lm_damping(hii, scale[6 * slot + i], radius, mind, maxd) * dp[i] * dp[i];
        st += dp[i] * dp[i];
      }
    }
    const Q4 qn = qnormalized(qmul(q, so3_exp(v3(dp[0], dp[1], dp[2]))));
    cand.q[4 * v] = qn.x; cand.q[4 * v + 1] = qn.y; cand.q[4 * v + 2] = qn.z; cand.q[4 * v + 3] = qn.w;
    cand.c[3 * v] = c.x + dp[3]; cand.c[3 * v + 1] = c.y + dp[4]; cand.c[3 * v + 2] = c.z + dp[5];
    xs = 1.0 + dot(c, c);
  }
  gd = wsum(gd); dd = wsum(dd); st = wsum(st); xs = wsum(xs);
  if (lane == 0) { atomicAdd(&scal[CC_G_DELTA], gd); atomicAdd(&scal[CC_D_DELTA], dd); atomicAdd(&scal[CC_STEP_SQ], st); atomicAdd(&scal[CC_X_SQ], xs); }
}

}  // namespace

void launch_camcal_accumulate(const CamCalProblem& Q, const CamCalState& S, bool with_jacobian, double* blocks, double* sys, double* cost_out, double* view_err, cudaStream_t st) {
  if (Q.n_active <= 0) return;
  const int grid = (Q.n_active + 3) / 4;
  if (with_jacobian) camcal_accumulate_kernel<true><<<grid, 128, 0, st>>>(Q, S, blocks, sys, nullptr, nullptr);
  else camcal_accumulate_kernel<false><<<grid, 128, 0, st>>>(Q, S, nullptr, nullptr, cost_out, view_err);
  count_launch();
}

void launch_camcal_step(const CamCalProblem& Q, const CamCalState& cur, const CamCalState& cand, const double* blocks, const double* sys, double* red, double* Y,
                        double* scale, int compute_scale, double radius, double min_diag, double max_diag, double* dk, double* scal, cudaStream_t st) {
  if (Q.n_active <= 0) return;
  const int grid = (Q.n_active + 127) / 128;
  camcal_reduce_kernel<<<(Q.n_active + RED_THREADS - 1) / RED_THREADS, RED_THREADS, 0, st>>>(Q, blocks, red, Y, scale, compute_scale, radius, min_diag, max_diag, scal);
  count_launch();
  camcal_solve_kernel<<<1, 32, 0, st>>>(Q, cur, cand, sys, red, scale + 6 * (size_t)Q.n_active, compute_scale, radius, min_diag, max_diag, dk, scal);
  count_launch();
  camcal_update_kernel<<<grid, 128, 0, st>>>(Q, cur, cand, blocks, Y, dk, scale, radius, min_diag, max_diag, scal);
  count_launch();
}

}  // namespace icc
