// SplineOptimFlags::POINTS: the board points as parameter blocks of the spline problem.
//
// Reference: SplineTrajectoryEstimator::SetFixedParams (core/spline_trajectory_estimator.impl.h:136-152) frees the homogeneous 4-vector of
// every track a view sees and gives it ceres::HomogeneousVectorParameterization(4) (Ceres 2.1 local_parameterization.cc, restated: Householder
// vector v, beta with (I - beta v v^T) x = |x| e_4; tangent Jacobian = |x| / 2 x the first three columns of H; Plus(x, d) = |x| H [sin(|d|/2) d/|d| ;
// cos(|d|/2)]).  The hot CLI never sets the flag, so this path is built for correctness, not for the roofline:
//   * the evaluation kernels stay as they are (they read the de-homogenised points of the state and treat them as constants);
//   * points_jac_kernel adds the blocks that involve the 3 C point columns (border columns of the normal equations): per corner the 2 x 3
//     tangent rows p = [m_t / w, -(m_t . X) / w] J_lp -- the residual depends on the point through X = x / w exactly like on the spline position
//     with the opposite sign, m_t being the translation covector the rows already carry -- and their products with the other 43 columns;
//   * points_update_kernel applies Plus and refreshes the de-homogenised copy and the local Jacobians of the candidate state.
#include "icc_kernels.h"
#include "icc_tile_common.cuh"
#include "icc_vision_rows.cuh"
#include "icc_points_math.cuh"

namespace icc {

namespace {

// de-homogenised point + local Jacobian (row-major 4 x 3) of one board point (icc_points_math.cuh)
ICC_D void prepare_point(const double4 x, double4* board, double* jac12) {
  const double xv[4] = {x.x, x.y, x.z, x.w};
  double b4[4];
  points_prepare(xv, b4, jac12);
  *board = make_double4(b4[0], b4[1], b4[2], b4[3]);
}

__global__ void points_prepare_kernel(int n, const double4* __restrict__ pts, double4* board, double* jac) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) prepare_point(pts[i], board + i, jac + 12 * i);
}

// candidate points = Plus(current, delta); squared ambient step / state norms are added to the LM scalars
__global__ void points_update_kernel(int n, int col_pts, const double4* __restrict__ cur, double4* cand, double4* board, double* jac, const double* __restrict__ delta, double* scal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double step = 0.0, xsq = 0.0;
  if (i < n) {
    const double4 x = cur[i];
    double4 o = x;
    if (col_pts >= 0) {
      const double d0 = delta[col_pts + 3 * i], d1 = delta[col_pts + 3 * i + 1], d2 = delta[col_pts + 3 * i + 2];
      const double xv[4] = {x.x, x.y, x.z, x.w}, dv[3] = {d0, d1, d2};
      double ov[4];
      points_plus(xv, dv, ov);
      o = make_double4(ov[0], ov[1], ov[2], ov[3]);
      step = (o.x - x.x) * (o.x - x.x) + (o.y - x.y) * (o.y - x.y) + (o.z - x.z) * (o.z - x.z) + (o.w - x.w) * (o.w - x.w);
      xsq = x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    }
    cand[i] = o;
    prepare_point(o, board + i, jac + 12 * i);
  }
  for (int off = 16; off > 0; off >>= 1) { step += __shfl_xor_sync(0xffffffffu, step, off); xsq += __shfl_xor_sync(0xffffffffu, xsq, off); }
  if ((threadIdx.x & 31) == 0 && col_pts >= 0 && (step != 0.0 || xsq != 0.0)) { atomicAdd(scal + SC_STEP_SQ, step); atomicAdd(scal + SC_X_SQ, xsq); }
}

ICC_D void ne_add_any(const NeLayout& L, int gi, int gj, double v) {
  const int lo = min(gi, gj), hi = max(gi, gj);
  double* dst;
  if (hi < L.nk) dst = L.ne + (int64_t)lo * L.ldb + (hi - lo);
  else if (lo < L.nk) dst = L.ne + L.off_E + (int64_t)lo * L.nb + (hi - L.nk);
  else dst = L.ne + L.off_C + (int64_t)(hi - L.nk) * L.nb + (lo - L.nk);
  atomicAdd(dst, v);
}

// one warp per frame: window staged once, one corner per lane; TAN: the rows of the tangent reprojection error
template <bool TAN>
__global__ void __launch_bounds__(128) points_jac_kernel(DeviceProblem P, DeviceState S, const double* __restrict__ pjac, int col_pts, TangentMeas T) {
  __shared__ FrameWin wins[4];
  __shared__ VisConst K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < MAX_INTR) K.intr[threadIdx.x] = S.glob[G_CAM_INTR + threadIdx.x];
  if (threadIdx.x == 32) {
    const Q4 q_ic = q4(S.glob[G_TIC + 0], S.glob[G_TIC + 1], S.glob[G_TIC + 2], S.glob[G_TIC + 3]);
    K.Ric = qmat(q_ic); K.tic = v3(S.glob[G_TIC + 4], S.glob[G_TIC + 5], S.glob[G_TIC + 6]);
    K.ld = S.glob[G_LD]; K.model = P.model; K.fov = P.dispatch_fov;
  }
  __syncthreads();
  NeLayout L; L.ne = P.ne; L.off_E = P.ne_off_E; L.off_C = P.ne_off_C; L.off_g = P.ne_off_g; L.off_cost = P.ne_off_cost; L.nk = P.nk; L.nb = P.nb; L.ldb = P.ldb;
  FrameWin& W = wins[warp];
  for (int f = blockIdx.x * 4 + warp; f < P.n_frames; f += gridDim.x * 4) {
    const int s_so3 = P.f_s_so3[f], s_r3 = P.f_s_r3[f];
    __syncwarp();
    {
      double4 k = make_double4(0, 0, 0, 1);
      if (lane < 6) k = S.so3[s_so3 + lane];
      const Q4 qa = q4(k.x, k.y, k.z, k.w);
      const Q4 qb = q4(__shfl_down_sync(0xffffffffu, k.x, 1), __shfl_down_sync(0xffffffffu, k.y, 1), __shfl_down_sync(0xffffffffu, k.z, 1), __shfl_down_sync(0xffffffffu, k.w, 1));
      if (lane < 5) stage_frame_increment(W, lane, qa, qb);
      if (lane == 0) { W.q0 = qa; W.u_so3 = P.f_u_so3[f]; W.u_r3 = P.f_u_r3[f]; }
      if (lane >= 8 && lane < 14) { const double4 p = S.r3[s_r3 + lane - 8]; W.p[lane - 8] = v3(p.x, p.y, p.z); }
    }
    __syncwarp();
    for (int c = P.f_off[f] + lane; c < P.f_off[f + 1]; c += 32) {
      const int pid = P.pid[c];
      const double2 ob = P.uv[c];
      const double4 X = P.board[pid];                                   // de-homogenised (w = 1)
      double row[2][44], yr[YR_N], r0, r1;
      if constexpr (TAN) vision_corner_rows<VIS_TANGENT>(W, K, v3(X.x, X.y, X.z), ob.y, T.bear[c], T.ok[c] != 0, T.s, row[0], 1, yr, r0, r1);
      else vision_corner_rows<-1>(W, K, v3(X.x, X.y, X.z), ob.x, ob.y, row[0], 1, yr, r0, r1);
      if (r0 == 1e10) continue;                                          // failed projection: zero Jacobian rows
      vision_yrow_expand(yr, row[1], 1);
      const double* J = pjac + 12 * pid;
      const double wh = S.pts[pid].w;                                    // homogeneous coordinate
      double p[2][3];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        // m_t = -(sum over the six R^3 knot columns): the basis coefficients sum to one
        double mt[3] = {0, 0, 0};
        for (int j = 0; j < 6; ++j) for (int k = 0; k < 3; ++k) mt[k] -= row[r][18 + 3 * j + k];
        const double a4[4] = {mt[0] / wh, mt[1] / wh, mt[2] / wh, -(mt[0] * X.x + mt[1] * X.y + mt[2] * X.z) / wh};   // d r / d (x, y, z, w)
        for (int i = 0; i < 3; ++i) p[r][i] = a4[0] * J[i] + a4[1] * J[3 + i] + a4[2] * J[6 + i] + a4[3] * J[9 + i];
      }
      const int gp = col_pts + 3 * pid;
      // point x point, gradient
      for (int a = 0; a < 3; ++a) {
        atomicAdd(L.ne + L.off_g + gp + a, p[0][a] * row[0][VIS_RES_COL] + p[1][a] * row[1][VIS_RES_COL]);
        for (int b = a; b < 3; ++b) ne_add_any(L, gp + a, gp + b, p[0][a] * p[0][b] + p[1][a] * p[1][b]);
      }
      // point x every other active column of the rows
      for (int cc = 0; cc < VIS_RES_COL; ++cc) {
        int g = -1;
        if (cc < 18) { const int b = P.so3_col[s_so3 + cc / 3]; g = b < 0 ? -1 : b + cc % 3; }
        else if (cc < 36) { const int b = P.r3_col[s_r3 + (cc - 18) / 3]; g = b < 0 ? -1 : b + (cc - 18) % 3; }
        else if (cc < 42) g = P.col_tic < 0 ? -1 : P.col_tic + (cc - 36);
        else g = P.col_ld;
        if (g < 0) continue;
        for (int a = 0; a < 3; ++a) ne_add_any(L, g, gp + a, row[0][cc] * p[0][a] + row[1][cc] * p[1][a]);
      }
    }
  }
}

}  // namespace

void launch_points_prepare(int n, const double4* pts, double4* board, double* jac, cudaStream_t st) {
  if (n <= 0) return;
  points_prepare_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, pts, board, jac); count_launch();
}
void launch_points_update(int n, int col_pts, const double4* cur, double4* cand, double4* board, double* jac, const double* delta, double* scal, cudaStream_t st) {
  if (n <= 0) return;
  points_update_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, col_pts, cur, cand, board, jac, delta, scal); count_launch();
}
void launch_points_jac(const DeviceProblem& P_in, const DeviceState& S, const double* pjac, int col_pts, int sm_count, cudaStream_t st, const TangentMeas* tan) {
  if (P_in.n_frames <= 0 || col_pts < 0) return;
  DeviceProblem P = P_in; P.board = S.board;
  int grid = (P.n_frames + 3) / 4; if (grid > 8 * sm_count) grid = 8 * sm_count;
  if (tan) points_jac_kernel<true><<<grid, 128, 0, st>>>(P, S, pjac, col_pts, *tan);
  else points_jac_kernel<false><<<grid, 128, 0, st>>>(P, S, pjac, col_pts, TangentMeas{nullptr, nullptr, 0.0});
  count_launch();
}

}  // namespace icc
