// Per-view board pose estimation (sm_90a): the step that fills the pose dataset the hot CLI consumes (SURVEY.md §8(f) row f1).
//
// Replaces, for every view in parallel, what the reference runs serially on the CPU in
//   PoseEstimator::EstimatePosesFromJson      src/core/pose_estimator.cc:92-191
//   PoseEstimator::EstimatePosePinhole        src/core/pose_estimator.cc:54-90
// i.e. theia::Camera::PixelToNormalizedCoordinates per corner, a calibrated absolute pose (RANSAC PnP, squared normalised
// reprojection error threshold, >= 6 inliers) and theia::BundleAdjustView (pose-only, Huber 1.345) on the inliers.
//
// Mapping to the machine: kernel 1 un-projects one corner per thread by Gauss-Newton on the forward model (the closed-form
// 2x3 projection Jacobians of icc_camera.cuh; one code path for all seven camera models, residual < 1e-13 px); kernel 2 gives
// one WARP per view: lanes stride over the corners, the 8x8 (homography) and 6x6 (pose) normal equations are reduced with warp
// shuffles and solved redundantly in registers by every lane (no shared memory, no divergence).  The calibration board is
// planar, so the initial pose comes from the normalised DLT homography; the refinement minimises the same cost as the
// reference's BundleAdjustView (normalised pinhole reprojection error, Huber 1.345) with Levenberg-Marquardt to a tighter
// tolerance than Ceres' defaults, so both land on the same optimum.
//
// Opt-in wide-angle residual (ICC_POSE_ERROR_TANGENT): corners are unit bearings (icc_bearing_math.cuh) and the same kernels minimise the
// local tangent reprojection error instead, so rays 90 degrees or more off the axis keep their views.  The residual is a template parameter
// chosen by the measurement type (double2 = normalised point, double4 = bearing); the default kernels compile to the same code as before.
//
// Opt-in rolling shutter (icc_set_pose_rolling_shutter): after the global-shutter pass, two more refinement-only passes score each corner
// against the pose at its row time (icc_rolling_shutter_math.cuh), with each view's velocities taken from its neighbours in time by a small
// kernel before each pass.  Rolling shutter is a template parameter of board_pose_kernel and point_refine_kernel; false is the code as before.
#include "icc_bearing_math.cuh"
#include "icc_camera.cuh"
#include "icc_host.h"
#include "icc_reduce.cuh"
#include "icc_rolling_shutter_math.cuh"
#include "icc_small_linalg.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>
#include <type_traits>

namespace icc {

namespace {

struct Intr { double k[MAX_INTR]; };

__global__ void unproject_kernel(int model, Intr K, int n, const double2* __restrict__ uv, double2* __restrict__ xy, int* __restrict__ ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double x = 0.0, y = 0.0;
  const bool good = unproject_gn(model, K.k, uv[i].x, uv[i].y, x, y);
  xy[i] = make_double2(x, y);
  if (ok) ok[i] = good ? 1 : 0;
}

__global__ void bearing_kernel(int model, Intr K, int n, const double2* __restrict__ uv, double4* __restrict__ b, int* __restrict__ ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  V3 r;
  const bool good = unproject_bearing(model, K.k, uv[i].x, uv[i].y, r);
  b[i] = make_double4(r.x, r.y, r.z, 0.0);
  if (ok) ok[i] = good ? 1 : 0;
}

// One Gauss-Newton system of the pose-only bundle adjustment over the masked corners of this view:
//   r = pi(R X + t) - x_n,  R <- R exp(delta) (right increment), t <- t + dt;  Huber(1.345) on |r| as in ba_options_ (:44-46)
struct PoseSys { double H[6][6]; double g[6]; double cost; };
ICC_D void pose_system(const PoseProblem& Q, const double2* xy, const unsigned char* use, int c0, int c1, double zref, Q4 q, V3 t, PoseSys& S, bool with_jacobian) {
  const int lane = threadIdx.x & 31;
  double H[21], g[6], cost = 0.0;
#pragma unroll
  for (int i = 0; i < 21; ++i) H[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  const double hub = 1.345;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    const V3 X = v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w - zref);
    const V3 RX = qrot(q, X), Pc = RX + t;
    const double iz = 1.0 / Pc.z, u = Pc.x * iz, v = Pc.y * iz;
    const double r0 = u - xy[c].x, r1 = v - xy[c].y, rn = sqrt(r0 * r0 + r1 * r1);
    // Huber: rho(s) = s for s <= a^2, 2 a sqrt(s) - a^2 beyond; cost = 1/2 rho(|r|^2); IRLS weight = rho'
    const double w = rn <= hub ? 1.0 : hub / rn;
    cost += rn <= hub ? 0.5 * rn * rn : hub * rn - 0.5 * hub * hub;
    if (!with_jacobian || !(Pc.z > 0.0)) { if (!(Pc.z > 0.0)) cost += 1e6; continue; }
    // d pi / d Pc rows, then d Pc / d(delta, t) = [-R [X]x | I]  ->  row_delta = -(row R) x X ... = X x (R^T row)
    const V3 a0 = v3(iz, 0.0, -u * iz), a1 = v3(0.0, iz, -v * iz);
    const V3 b0 = cross(X, qrot_inv(q, a0)), b1 = cross(X, qrot_inv(q, a1));
    const double J0[6] = {b0.x, b0.y, b0.z, a0.x, a0.y, a0.z}, J1[6] = {b1.x, b1.y, b1.z, a1.x, a1.y, a1.z};
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      g[i] += w * (J0[i] * r0 + J1[i] * r1);
#pragma unroll
      for (int j = 0; j <= i; ++j) { H[idx] += w * (J0[i] * J0[j] + J1[i] * J1[j]); ++idx; }
    }
  }
  S.cost = warp_sum(cost);
  if (!with_jacobian) return;
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    S.g[i] = warp_sum(g[i]);
#pragma unroll
    for (int j = 0; j <= i; ++j) { const double v = warp_sum(H[idx]); S.H[i][j] = v; S.H[j][i] = v; ++idx; }
  }
}

// The same system for the tangent residual against bearings (icc_bearing_math.cuh): r = (e1.d, e2.d) / (b.d), d = R X + t; 1e6 where b.d <= 0.
// An overload rather than a shared body, so that the normalised system above keeps its code.
ICC_D void pose_system(const PoseProblem& Q, const double4* bear, const unsigned char* use, int c0, int c1, double zref, Q4 q, V3 t, PoseSys& S, bool with_jacobian) {
  const int lane = threadIdx.x & 31;
  double H[21], g[6], cost = 0.0;
#pragma unroll
  for (int i = 0; i < 21; ++i) H[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  const double hub = 1.345;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    const V3 X = v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w - zref);
    const V3 Pc = qrot(q, X) + t;
    const TangentErr E(Pc, v3(bear[c].x, bear[c].y, bear[c].z));
    const double r0 = E.r0, r1 = E.r1, rn = sqrt(r0 * r0 + r1 * r1);
    const double w = rn <= hub ? 1.0 : hub / rn;
    cost += rn <= hub ? 0.5 * rn * rn : hub * rn - 0.5 * hub * hub;
    if (!with_jacobian || !E.front()) { if (!E.front()) cost += 1e6; continue; }
    double J0[6], J1[6]; V3 P0, P1;
    tangent_jacobians(E, q, X, J0, J1, P0, P1);
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      g[i] += w * (J0[i] * r0 + J1[i] * r1);
#pragma unroll
      for (int j = 0; j <= i; ++j) { H[idx] += w * (J0[i] * J0[j] + J1[i] * J1[j]); ++idx; }
    }
  }
  S.cost = warp_sum(cost);
  if (!with_jacobian) return;
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    S.g[i] = warp_sum(g[i]);
#pragma unroll
    for (int j = 0; j <= i; ++j) { const double v = warp_sum(H[idx]); S.H[i][j] = v; S.H[j][i] = v; ++idx; }
  }
}

// the tangent error of one corner for the inlier and mean-error passes; false where b.d <= 0
ICC_D bool tangent_err(V3 Pc, double4 m, double& r0, double& r1) { const TangentErr E(Pc, v3(m.x, m.y, m.z)); r0 = E.r0; r1 = E.r1; return E.front(); }

// Rolling shutter: the per-corner row times (uv[c].y * line_delay) and this view's velocities
struct RsView { const double2* uv; double line_delay; RsMotion m; };

// The system of either residual with every corner at its row time (rs_pose_residual); 1e6 where the point is behind the measurement
template <class M>
ICC_D void pose_system_rs(const PoseProblem& Q, const M* meas, const unsigned char* use, int c0, int c1, double zref, Q4 q, V3 t, const RsView& rs, PoseSys& S, bool with_jacobian) {
  const int lane = threadIdx.x & 31;
  double H[21], g[6], cost = 0.0;
#pragma unroll
  for (int i = 0; i < 21; ++i) H[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) g[i] = 0.0;
  const double hub = 1.345;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    const V3 X = v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w - zref);
    double r0, r1, J0[6], J1[6];
    const bool front = rs_pose_residual(meas[c], q, t, X, rs.m, rs.uv[c].y * rs.line_delay, r0, r1, J0, J1);
    const double rn = sqrt(r0 * r0 + r1 * r1);
    const double w = rn <= hub ? 1.0 : hub / rn;
    cost += rn <= hub ? 0.5 * rn * rn : hub * rn - 0.5 * hub * hub;
    if (!with_jacobian || !front) { if (!front) cost += 1e6; continue; }
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      g[i] += w * (J0[i] * r0 + J1[i] * r1);
#pragma unroll
      for (int j = 0; j <= i; ++j) { H[idx] += w * (J0[i] * J0[j] + J1[i] * J1[j]); ++idx; }
    }
  }
  S.cost = warp_sum(cost);
  if (!with_jacobian) return;
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    S.g[i] = warp_sum(g[i]);
#pragma unroll
    for (int j = 0; j <= i; ++j) { const double v = warp_sum(H[idx]); S.H[i][j] = v; S.H[j][i] = v; ++idx; }
  }
}

// the system of the pose refinement: global shutter (pose_system) or rolling shutter (pose_system_rs)
template <bool RS, class M>
ICC_D void view_system(const PoseProblem& Q, const M* xy, const unsigned char* use, int c0, int c1, double zref, Q4 q, V3 t, const RsView& rs, PoseSys& S, bool with_jacobian) {
  if constexpr (RS) pose_system_rs(Q, xy, use, c0, c1, zref, q, t, rs, S, with_jacobian);
  else pose_system(Q, xy, use, c0, c1, zref, q, t, S, with_jacobian);
}

// Levenberg-Marquardt on the 6 pose parameters (all lanes run the identical scalar logic on warp-reduced sums)
template <class M, bool RS = false>
ICC_D void pose_refine(const PoseProblem& Q, const M* xy, const unsigned char* use, int c0, int c1, double zref, Q4& q, V3& t, const RsView& rs) {
  PoseSys S;
  view_system<RS>(Q, xy, use, c0, c1, zref, q, t, rs, S, true);
  double lambda = 1e-4, cost = S.cost;
  for (int it = 0; it < 50; ++it) {
    double A[6][6], b[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      b[i] = -S.g[i];
#pragma unroll
      for (int j = 0; j < 6; ++j) A[i][j] = S.H[i][j];
      A[i][i] += lambda * (S.H[i][i] + 1e-12);
    }
    if (!chol_solve<6>(A, b)) { lambda *= 10.0; if (lambda > 1e12) break; continue; }
    const Q4 qn = qnormalized(qmul(q, so3_exp(v3(b[0], b[1], b[2]))));
    const V3 tn = t + v3(b[3], b[4], b[5]);
    PoseSys Sn;
    view_system<RS>(Q, xy, use, c0, c1, zref, qn, tn, rs, Sn, false);
    const double step2 = b[0] * b[0] + b[1] * b[1] + b[2] * b[2] + b[3] * b[3] + b[4] * b[4] + b[5] * b[5];
    if (Sn.cost < cost) {
      const double dec = cost - Sn.cost;
      q = qn; t = tn; cost = Sn.cost; lambda = fmax(lambda * 0.1, 1e-12);
      if (dec <= (Q.lm_rel_tol > 0.0 ? Q.lm_rel_tol : 1e-15) * cost || step2 < 1e-28) break;
      view_system<RS>(Q, xy, use, c0, c1, zref, q, t, rs, S, true);
    } else {
      if (step2 < 1e-28) break;
      lambda *= 10.0;
      if (lambda > 1e12) break;
    }
  }
}

// Normalised DLT homography board plane -> image of one view, by one warp (every lane returns the same values):
// marks the usable corners in use[], returns their count n, the board plane height zref and H (row-major, acting on
// (X, Y, 1) with Z = zref); false = too few corners / degenerate / non-planar target.
ICC_D bool board_homography(const PoseProblem& Q, const double2* __restrict__ xy, const int* __restrict__ okc, unsigned char* __restrict__ use, int c0, int c1,
                            double& n_out, double& zref_out, double (&Hm)[9]) {
  const int lane = threadIdx.x & 31;
  // ---- usable corners, board plane, Hartley normalisation ------------------------------------------------------------------
  double n = 0.0, sX = 0.0, sY = 0.0, sZ = 0.0, sx = 0.0, sy = 0.0;
  for (int c = c0 + lane; c < c1; c += 32) {
    const int id = Q.pid[c];
    const bool u = (okc == nullptr || okc[c] != 0) && id >= 0 && id < Q.n_points;
    use[c] = u ? 1 : 0;
    if (!u) continue;
    const double4 Xb = Q.board[id];
    n += 1.0; sX += Xb.x / Xb.w; sY += Xb.y / Xb.w; sZ += Xb.z / Xb.w; sx += xy[c].x; sy += xy[c].y;
  }
  n = warp_sum(n); sX = warp_sum(sX); sY = warp_sum(sY); sZ = warp_sum(sZ); sx = warp_sum(sx); sy = warp_sum(sy);
  __syncwarp();
  n_out = n;
  if (c1 - c0 < Q.min_points || n < 6.0) return false;   // pose_estimator.cc:140 (all corners counted), :65
  const double mX = sX / n, mY = sY / n, zref = sZ / n, mx = sx / n, my = sy / n;
  zref_out = zref;
  double dB = 0.0, dI = 0.0, dz = 0.0;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    const double X = Xb.x / Xb.w - mX, Y = Xb.y / Xb.w - mY, x = xy[c].x - mx, y = xy[c].y - my;
    dB += sqrt(X * X + Y * Y); dI += sqrt(x * x + y * y); dz = fmax(dz, fabs(Xb.z / Xb.w - zref));
  }
  dB = warp_sum(dB) / n; dI = warp_sum(dI) / n;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dz = fmax(dz, __shfl_xor_sync(0xffffffffu, dz, o));
  if (!(dB > 0.0) || !(dI > 0.0) || dz > 0.05 * dB) return false;   // degenerate, or too far from a plane for the homography to start the refinement
                                                                     // (a few per cent of the board size -- refined board points of a printed target -- are fine: pose_system uses the real 3-D points)
  const double sB = sqrt(2.0) / dB, sI = sqrt(2.0) / dI;
  // ---- homography (h33 = 1) from the normal equations of the DLT rows -------------------------------------------------------
  double M[36], v8[8];
#pragma unroll
  for (int i = 0; i < 36; ++i) M[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) v8[i] = 0.0;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    const double X = (Xb.x / Xb.w - mX) * sB, Y = (Xb.y / Xb.w - mY) * sB, x = (xy[c].x - mx) * sI, y = (xy[c].y - my) * sI;
    const double ra[8] = {X, Y, 1.0, 0.0, 0.0, 0.0, -x * X, -x * Y}, rb[8] = {0.0, 0.0, 0.0, X, Y, 1.0, -y * X, -y * Y};
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v8[i] += ra[i] * x + rb[i] * y;
#pragma unroll
      for (int j = 0; j <= i; ++j) { M[idx] += ra[i] * ra[j] + rb[i] * rb[j]; ++idx; }
    }
  }
  double A8[8][8], h[8];
  {
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      h[i] = warp_sum(v8[i]);
#pragma unroll
      for (int j = 0; j <= i; ++j) { const double v = warp_sum(M[idx]); A8[i][j] = v; A8[j][i] = v; ++idx; }
    }
  }
  if (!chol_solve<8>(A8, h)) return false;
  // de-normalise: H = T_img^-1 Hn T_board,  T_board = [sB 0 -sB mX; 0 sB -sB mY; 0 0 1],  T_img^-1 = [1/sI 0 mx; 0 1/sI my; 0 0 1]
  double Hn[9] = {h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7], 1.0}, G[9];
#pragma unroll
  for (int r = 0; r < 3; ++r) { G[3 * r] = Hn[3 * r] * sB; G[3 * r + 1] = Hn[3 * r + 1] * sB; G[3 * r + 2] = Hn[3 * r + 2] - sB * (Hn[3 * r] * mX + Hn[3 * r + 1] * mY); }
#pragma unroll
  for (int cidx = 0; cidx < 3; ++cidx) { Hm[cidx] = G[cidx] / sI + mx * G[6 + cidx]; Hm[3 + cidx] = G[3 + cidx] / sI + my * G[6 + cidx]; Hm[6 + cidx] = G[6 + cidx]; }
  return true;
}

// H ~ [r1 r2 t] (points on the plane z = zref, shifted to z = 0): scale, cheirality, Gram-Schmidt -> R_cw, t
ICC_D void pose_from_homography(const double (&Hm)[9], Q4& q, V3& t) {
  V3 h1 = v3(Hm[0], Hm[3], Hm[6]), h2 = v3(Hm[1], Hm[4], Hm[7]), h3 = v3(Hm[2], Hm[5], Hm[8]);
  double s = 2.0 / (sqrt(dot(h1, h1)) + sqrt(dot(h2, h2)));
  if (h3.z * s < 0.0) s = -s;
  V3 r1 = s * h1, r2 = s * h2;
  t = s * h3;
  r1 = (1.0 / sqrt(dot(r1, r1))) * r1;
  r2 = r2 - dot(r1, r2) * r1; r2 = (1.0 / sqrt(dot(r2, r2))) * r2;
  const V3 r3 = cross(r1, r2);
  q = quat_from_columns(r1, r2, r3);          // R_cw
}

// Start of a view from bearings: rotate them so that their normalised mean is +z (rows e1, e2, m of R_m), take the homography of those
// within ~80 degrees of the mean on that frame's normalised plane (xy_h, ok_h: per-corner scratch), rotate the pose back.  Every usable
// corner, those beyond 80 degrees included, is marked in use[] for the refinement.
ICC_D bool bearing_start(const PoseProblem& Q, const double4* bear, const int* okc, unsigned char* use, double2* xy_h, int* ok_h, int c0, int c1, double& n, double& zref, Q4& q, V3& t) {
  const int lane = threadIdx.x & 31;
  V3 m = v3(0.0, 0.0, 0.0);
  for (int c = c0 + lane; c < c1; c += 32) {
    const int id = Q.pid[c];
    if (okc[c] != 0 && id >= 0 && id < Q.n_points) m = m + v3(bear[c].x, bear[c].y, bear[c].z);
  }
  m = v3(warp_sum(m.x), warp_sum(m.y), warp_sum(m.z));
  const double mn = sqrt(dot(m, m));
  m = mn > 0.0 ? (1.0 / mn) * m : v3(0.0, 0.0, 1.0);
  V3 e1, e2; tangent_basis(m, e1, e2);
  const double cos_max = 0.17364817766693033;   // cos(80 degrees)
  for (int c = c0 + lane; c < c1; c += 32) {
    const V3 b = v3(bear[c].x, bear[c].y, bear[c].z), bm = v3(dot(e1, b), dot(e2, b), dot(m, b));
    const bool near = bm.z > cos_max;
    ok_h[c] = okc[c] != 0 && near ? 1 : 0;
    xy_h[c] = near ? make_double2(bm.x / bm.z, bm.y / bm.z) : make_double2(0.0, 0.0);
  }
  __syncwarp();
  double Hm[9];
  if (!board_homography(Q, xy_h, ok_h, use, c0, c1, n, zref, Hm)) return false;
  Q4 qm; V3 tm;
  pose_from_homography(Hm, qm, tm);
  const Q4 rm_t = quat_from_columns(e1, e2, m);   // R_m^T
  q = qnormalized(qmul(rm_t, qm)); t = qrot(rm_t, tm);
  for (int c = c0 + lane; c < c1; c += 32) {
    const int id = Q.pid[c];
    use[c] = okc[c] != 0 && id >= 0 && id < Q.n_points ? 1 : 0;
  }
  __syncwarp();
  return true;
}

// M = double2: normalised points (the reference's residual); M = double4: bearings, the tangent residual (xy_h / ok_h: per-corner scratch of the
// start).  The normalised branches keep their own text, so that board_pose_kernel<double2> compiles to the same code as the pre-template kernel.
// RS (refinement-only passes): every corner at its row time uv[c].y * line_delay, with the view's velocities vel[6f..6f+5] = (w, u).
template <class M, bool RS = false>
__global__ void __launch_bounds__(128) board_pose_kernel(PoseProblem Q, const M* __restrict__ xy, const int* __restrict__ okc, unsigned char* __restrict__ use,
                                                        double* q_out, double* p_out, double* __restrict__ err_out, int* valid_out, double2* __restrict__ xy_h, int* __restrict__ ok_h,
                                                        RsPass rsp) {
  constexpr bool kTangent = std::is_same<M, double4>::value;
  const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (f >= Q.n_frames) return;
  const int c0 = Q.f_off[f], c1 = Q.f_off[f + 1];
  auto fail = [&]() {
    if (lane == 0) { q_out[4 * f] = 0.0; q_out[4 * f + 1] = 0.0; q_out[4 * f + 2] = 0.0; q_out[4 * f + 3] = 1.0; p_out[3 * f] = 0.0; p_out[3 * f + 1] = 0.0; p_out[3 * f + 2] = 0.0; err_out[f] = 0.0; valid_out[f] = 0; }
  };
  double n = 0.0, zref = 0.0;
  Q4 q; V3 t;
  RsView rs;
  if constexpr (RS) {
    const double* v = rsp.vel + 6 * f;
    rs.uv = rsp.uv; rs.line_delay = rsp.line_delay; rs.m.w = v3(v[0], v[1], v[2]); rs.m.u = v3(v[3], v[4], v[5]);
  }
  if (Q.refine_only) {
    // PoseEstimator::OptimizeAllPoses (pose_estimator.cc:226-236): BundleAdjustView again from the stored pose -- no homography, so the
    // board may have left its plane (optimised board points); views that were dropped stay dropped and keep their outputs
    if (!valid_out[f]) return;
    for (int c = c0 + lane; c < c1; c += 32) {
      const int id = Q.pid[c];
      const bool u = okc[c] != 0 && id >= 0 && id < Q.n_points;
      use[c] = u ? 1 : 0;
      if (u) n += 1.0;
    }
    n = warp_sum(n);
    __syncwarp();
    if (c1 - c0 < Q.min_points || n < 6.0) { fail(); return; }
    const Q4 qw = qnormalized(q4(q_out[4 * f], q_out[4 * f + 1], q_out[4 * f + 2], q_out[4 * f + 3]));
    q = qconj(qw);
    t = -qrot(q, v3(p_out[3 * f], p_out[3 * f + 1], p_out[3 * f + 2]));
  } else {
    if constexpr (kTangent) {
      if (!bearing_start(Q, xy, okc, use, xy_h, ok_h, c0, c1, n, zref, q, t)) { fail(); return; }
    } else {
      double Hm[9];
      if (!board_homography(Q, xy, okc, use, c0, c1, n, zref, Hm)) { fail(); return; }
      // H ~ [r1 r2 t] (points on the plane z = zref, shifted to z = 0): scale, cheirality, Gram-Schmidt
      V3 h1 = v3(Hm[0], Hm[3], Hm[6]), h2 = v3(Hm[1], Hm[4], Hm[7]), h3 = v3(Hm[2], Hm[5], Hm[8]);
      double s = 2.0 / (sqrt(dot(h1, h1)) + sqrt(dot(h2, h2)));
      if (h3.z * s < 0.0) s = -s;
      V3 r1 = s * h1, r2 = s * h2;
      t = s * h3;
      r1 = (1.0 / sqrt(dot(r1, r1))) * r1;
      r2 = r2 - dot(r1, r2) * r1; r2 = (1.0 / sqrt(dot(r2, r2))) * r2;
      const V3 r3 = cross(r1, r2);
      q = quat_from_columns(r1, r2, r3);          // R_cw
    }
  }
  // ---- refinement, inlier selection with the reference's squared normalised threshold, refinement on the inliers -------------
  pose_refine<M, RS>(Q, xy, use, c0, c1, zref, q, t, rs);
  double n_in = 0.0, n_out = 0.0;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    V3 Pc = qrot(q, v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w - zref)) + t;
    if constexpr (RS) { const double tau = rs.uv[c].y * rs.line_delay; Pc = rs_point(rs_rotation(rs.m, tau), rs.m, tau, Pc); }
    bool in;
    if constexpr (kTangent) {
      double r0, r1e;
      in = tangent_err(Pc, xy[c], r0, r1e) && r0 * r0 + r1e * r1e < Q.thresh_sq;
    } else {
      const double r0 = Pc.x / Pc.z - xy[c].x, r1e = Pc.y / Pc.z - xy[c].y;
      in = Pc.z > 0.0 && r0 * r0 + r1e * r1e < Q.thresh_sq;
    }
    if (in) n_in += 1.0; else { n_out += 1.0; use[c] = 0; }
  }
  n_in = warp_sum(n_in); n_out = warp_sum(n_out);
  __syncwarp();
  if (n_in < 6.0) { fail(); return; }
  if (n_out > 0.0) pose_refine<M, RS>(Q, xy, use, c0, c1, zref, q, t, rs);
  // ---- mean reprojection error of the kept observations (:164-181; the view camera is the unit pinhole) ----------------------
  double e = 0.0;
  for (int c = c0 + lane; c < c1; c += 32) {
    if (!use[c]) continue;
    const double4 Xb = Q.board[Q.pid[c]];
    V3 Pc = qrot(q, v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w - zref)) + t;
    if constexpr (RS) { const double tau = rs.uv[c].y * rs.line_delay; Pc = rs_point(rs_rotation(rs.m, tau), rs.m, tau, Pc); }
    if constexpr (kTangent) {
      double r0, r1e;
      tangent_err(Pc, xy[c], r0, r1e);
      e += sqrt(r0 * r0 + r1e * r1e);
    } else {
      const double r0 = Pc.x / Pc.z - xy[c].x, r1e = Pc.y / Pc.z - xy[c].y;
      e += sqrt(r0 * r0 + r1e * r1e);
    }
  }
  e = warp_sum(e) / n_in;
  if (lane == 0) {
    // undo the plane shift: Pc = R (X - zref e_z) + t  =>  t_full = t - zref R e_z ; camera centre p_wc = -R^T t_full ; q_wc = q^*
    const V3 tf = t - zref * qrot(q, v3(0.0, 0.0, 1.0));
    const V3 pw = -qrot_inv(q, tf);
    const Q4 qw = qconj(q);
    const bool keep = e <= Q.max_err;
    q_out[4 * f] = qw.x; q_out[4 * f + 1] = qw.y; q_out[4 * f + 2] = qw.z; q_out[4 * f + 3] = qw.w;
    p_out[3 * f] = pw.x; p_out[3 * f + 1] = pw.y; p_out[3 * f + 2] = pw.z;
    err_out[f] = e; valid_out[f] = keep ? 1 : 0;
  }
}

// Focal length of a view from its board homography on principal-point-centred pixels (square pixels, zero skew):
// H ~ K [r1 r2 t], K = diag(f, f, 1), r1 . r2 = 0 and |r1| = |r2| give two linear equations a_i + f^2 b_i = 0 (Zhang's
// constraints); least squares over both.  f2_out[v] = f^2, or 0 when the view is unusable / the estimate is not positive.
__global__ void __launch_bounds__(128) board_focal_kernel(PoseProblem Q, const double2* __restrict__ uv, double cx, double cy, double2* __restrict__ xy,
                                                         unsigned char* __restrict__ use, double* __restrict__ f2_out) {
  const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (f >= Q.n_frames) return;
  const int c0 = Q.f_off[f], c1 = Q.f_off[f + 1];
  for (int c = c0 + lane; c < c1; c += 32) xy[c] = make_double2(uv[c].x - cx, uv[c].y - cy);
  __syncwarp();
  double n = 0.0, zref = 0.0, H[9], f2 = 0.0;
  if (board_homography(Q, xy, nullptr, use, c0, c1, n, zref, H)) {
    const double a1 = H[0] * H[1] + H[3] * H[4], b1 = H[6] * H[7];
    const double a2 = H[0] * H[0] + H[3] * H[3] - H[1] * H[1] - H[4] * H[4], b2 = H[6] * H[6] - H[7] * H[7];
    const double den = b1 * b1 + b2 * b2;
    if (den > 0.0) f2 = -(a1 * b1 + a2 * b2) / den;
    if (!(f2 > 0.0) || !isfinite(f2)) f2 = 0.0;
  }
  if (lane == 0) f2_out[f] = f2;
}

__global__ void pinhole_normalize_kernel(int n, const double2* __restrict__ uv, double cx, double cy, double inv_f, double2* __restrict__ xy, int* __restrict__ ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  xy[i] = make_double2((uv[i].x - cx) * inv_f, (uv[i].y - cy) * inv_f);
  ok[i] = 1;
}


// theia::BundleAdjustTracks with every camera constant (PoseEstimator::OptimizeBoardPoints, pose_estimator.cc:193-224; the tail of
// CameraCalibrator::RunCalibration, camera_calibrator.cc:207-216): with the cameras fixed every board point is its own 3-parameter
// problem, so ONE WARP owns one point: lanes stride over the point's observations (CSR by point, built on the host), the 3x3
// Levenberg-Marquardt system is warp-reduced and solved in registers by every lane.  Residual: Huber(1.345) on
//   normalised == 1 :  (R_cw (X - c)).xy / z - x_n          (the pose estimator's unit-pinhole views with undistorted features)
//   normalised == 0 :  CameraToPixelCoordinates(intr, R_cw (X - c)) - pixel     (the camera calibrator's views)
//   TANGENT         :  the tangent error of R_cw (X - c) against the corner's bearing  (the pose estimator's views in tangent mode)
//   RS (with normalised or TANGENT): the point at the corner's row time, exp(-tau [w]x) (R_cw (X - c) - tau u), rows A^T a as in pose_system_rs
struct PointSys { double H[3][3]; double g[3]; double cost; };
template <bool TANGENT, bool RS = false>
ICC_D void point_system(const PointProblem& Q, const double4* __restrict__ bear, int o0, int o1, V3 X, PointSys& S, bool with_jacobian, const RsPass& rsp) {
  const int lane = threadIdx.x & 31;
  double H[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0}, cost = 0.0;
  const double hub = Q.huber;
  for (int o = o0 + lane; o < o1; o += 32) {
    const int c = Q.pt_obs[o], v = Q.obs_view[c];
    const Q4 q = q4(Q.q_cw[4 * v], Q.q_cw[4 * v + 1], Q.q_cw[4 * v + 2], Q.q_cw[4 * v + 3]);
    V3 pc = qrot(q, X - v3(Q.cam_c[3 * v], Q.cam_c[3 * v + 1], Q.cam_c[3 * v + 2]));
    [[maybe_unused]] Q4 A;
    if constexpr (RS) {
      const double* vel = rsp.vel + 6 * v;
      RsMotion m; m.w = v3(vel[0], vel[1], vel[2]); m.u = v3(vel[3], vel[4], vel[5]);
      const double tau = rsp.uv[c].y * rsp.line_delay;
      A = rs_rotation(m, tau); pc = rs_point(A, m, tau, pc);
    }
    double r0, r1; V3 a0, a1;
    if constexpr (TANGENT) {
      const double4 m = bear[c];
      const TangentErr E(pc, v3(m.x, m.y, m.z));
      if (!E.front()) { cost += 1e6; continue; }
      r0 = E.r0; r1 = E.r1; E.rows(a0, a1);
    } else if (Q.normalized) {
      if (!(pc.z > 0.0)) { cost += 1e6; continue; }
      const double iz = 1.0 / pc.z, u = pc.x * iz, w = pc.y * iz;
      r0 = u - Q.meas[c].x; r1 = w - Q.meas[c].y;
      a0 = v3(iz, 0.0, -u * iz); a1 = v3(0.0, iz, -w * iz);
    } else {
      const Proj pr = project(Q.model, Q.intr, pc, true);
      if (!pr.ok) { cost += 1e10; continue; }
      r0 = pr.u - Q.meas[c].x; r1 = pr.v - Q.meas[c].y;
      a0 = v3(pr.J[0], pr.J[1], pr.J[2]); a1 = v3(pr.J[3], pr.J[4], pr.J[5]);
    }
    const double rn = sqrt(r0 * r0 + r1 * r1), wgt = rn <= hub ? 1.0 : hub / rn;
    cost += rn <= hub ? 0.5 * rn * rn : hub * rn - 0.5 * hub * hub;
    if (!with_jacobian) continue;
    if constexpr (RS) { a0 = qrot_inv(A, a0); a1 = qrot_inv(A, a1); }
    const V3 j0 = qrot_inv(q, a0), j1 = qrot_inv(q, a1);   // rows of J_proj R_cw
    g[0] += wgt * (j0.x * r0 + j1.x * r1); g[1] += wgt * (j0.y * r0 + j1.y * r1); g[2] += wgt * (j0.z * r0 + j1.z * r1);
    H[0] += wgt * (j0.x * j0.x + j1.x * j1.x); H[1] += wgt * (j0.x * j0.y + j1.x * j1.y); H[2] += wgt * (j0.x * j0.z + j1.x * j1.z);
    H[3] += wgt * (j0.y * j0.y + j1.y * j1.y); H[4] += wgt * (j0.y * j0.z + j1.y * j1.z); H[5] += wgt * (j0.z * j0.z + j1.z * j1.z);
  }
  S.cost = warp_sum(cost);
  if (!with_jacobian) return;
#pragma unroll
  for (int i = 0; i < 3; ++i) S.g[i] = warp_sum(g[i]);
  const double h0 = warp_sum(H[0]), h1 = warp_sum(H[1]), h2 = warp_sum(H[2]), h3 = warp_sum(H[3]), h4 = warp_sum(H[4]), h5 = warp_sum(H[5]);
  S.H[0][0] = h0; S.H[0][1] = h1; S.H[0][2] = h2; S.H[1][0] = h1; S.H[1][1] = h3; S.H[1][2] = h4; S.H[2][0] = h2; S.H[2][1] = h4; S.H[2][2] = h5;
}

// TANGENT: Q.meas is unused, the corners' bearings come in bear.  RS: the views' velocities and the corners' row times come in rsp.
template <bool TANGENT, bool RS = false>
__global__ void __launch_bounds__(128) point_refine_kernel(PointProblem Q, double4* __restrict__ board_out, int* __restrict__ optimized, const double4* __restrict__ bear, RsPass rsp) {
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= Q.n_points) return;
  const int o0 = Q.pt_off[p], o1 = Q.pt_off[p + 1];
  const double4 Xb = Q.board_in[p];
  if (o1 - o0 <= Q.min_obs) { if (lane == 0) { board_out[p] = Xb; optimized[p] = 0; } return; }   // pose_estimator.cc:202-206
  V3 X = v3(Xb.x / Xb.w, Xb.y / Xb.w, Xb.z / Xb.w);
  PointSys S;
  point_system<TANGENT, RS>(Q, bear, o0, o1, X, S, true, rsp);
  double lambda = 1e-4, cost = S.cost;
  for (int it = 0; it < 50; ++it) {
    double A[3][3], b[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      b[i] = -S.g[i];
#pragma unroll
      for (int j = 0; j < 3; ++j) A[i][j] = S.H[i][j];
      A[i][i] += lambda * (S.H[i][i] + 1e-12);
    }
    if (!chol_solve<3>(A, b)) { lambda *= 10.0; if (lambda > 1e12) break; continue; }
    const V3 Xn = X + v3(b[0], b[1], b[2]);
    PointSys Sn;
    point_system<TANGENT, RS>(Q, bear, o0, o1, Xn, Sn, false, rsp);
    const double step2 = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
    if (Sn.cost < cost) {
      const double dec = cost - Sn.cost;
      X = Xn; cost = Sn.cost; lambda = fmax(lambda * 0.1, 1e-12);
      if (dec <= 1e-15 * cost || step2 < 1e-30) break;
      point_system<TANGENT, RS>(Q, bear, o0, o1, X, S, true, rsp);
    } else {
      if (step2 < 1e-30) break;
      lambda *= 10.0;
      if (lambda > 1e12) break;
    }
  }
  if (lane == 0) { board_out[p] = make_double4(X.x, X.y, X.z, 1.0); optimized[p] = 1; }
}

// Velocities of every view from its neighbours in time, one thread per view over the time-sorted index order[] (times ts[], ascending).
// The neighbours are the nearest valid views before and after it at a positive gap of at most max_gap; both: central difference, one:
// one-sided between it and the view, none: w = u = 0 (the global-shutter model).  nbr[f] = number of neighbours used; -1 (and zero velocities)
// for an invalid view.
__global__ void view_velocity_kernel(int n, const int* __restrict__ order, const double* __restrict__ ts, double max_gap, const double* __restrict__ q_wc,
                                     const double* __restrict__ p_wc, const int* __restrict__ valid, double* __restrict__ vel, int* __restrict__ nbr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = order[i];
  const double tf = ts[i];
  int a = -1, b = -1;
  if (valid[f]) {
    for (int j = i - 1; j >= 0 && tf - ts[j] <= max_gap; --j) if (tf - ts[j] > 0.0 && valid[order[j]]) { a = j; break; }
    for (int j = i + 1; j < n && ts[j] - tf <= max_gap; ++j) if (ts[j] - tf > 0.0 && valid[order[j]]) { b = j; break; }
  }
  RsMotion m; m.w = v3(0.0, 0.0, 0.0); m.u = v3(0.0, 0.0, 0.0);
  if (a >= 0 || b >= 0) {
    const int fa = a >= 0 ? order[a] : f, fb = b >= 0 ? order[b] : f;
    auto qv = [&](int v) { return qnormalized(q4(q_wc[4 * v], q_wc[4 * v + 1], q_wc[4 * v + 2], q_wc[4 * v + 3])); };
    auto pv = [&](int v) { return v3(p_wc[3 * v], p_wc[3 * v + 1], p_wc[3 * v + 2]); };
    m = rs_view_velocity(qv(fa), pv(fa), a >= 0 ? ts[a] : tf, qv(fb), pv(fb), b >= 0 ? ts[b] : tf, qv(f));
  }
  double* o = vel + 6 * f;
  o[0] = m.w.x; o[1] = m.w.y; o[2] = m.w.z; o[3] = m.u.x; o[4] = m.u.y; o[5] = m.u.z;
  nbr[f] = valid[f] ? (a >= 0) + (b >= 0) : -1;
}

}  // namespace

void launch_unproject(int model, const double* intr, int n, const double2* uv, double2* xy, int* ok, cudaStream_t st) {
  if (n <= 0) return;
  Intr K; for (int i = 0; i < MAX_INTR; ++i) K.k[i] = intr[i];
  unproject_kernel<<<(n + 127) / 128, 128, 0, st>>>(model, K, n, uv, xy, ok);
  count_launch();
}

void launch_bearings(int model, const double* intr, int n, const double2* uv, double4* b, int* ok, cudaStream_t st) {
  if (n <= 0) return;
  Intr K; for (int i = 0; i < MAX_INTR; ++i) K.k[i] = intr[i];
  bearing_kernel<<<(n + 127) / 128, 128, 0, st>>>(model, K, n, uv, b, ok);
  count_launch();
}

void launch_board_poses(const PoseProblem& Q, const double2* xy, const int* ok, unsigned char* use, double* q_wc, double* p_wc, double* err, int* valid, cudaStream_t st) {
  if (Q.n_frames <= 0) return;
  board_pose_kernel<double2><<<(Q.n_frames + 3) / 4, 128, 0, st>>>(Q, xy, ok, use, q_wc, p_wc, err, valid, nullptr, nullptr, RsPass{});
  count_launch();
}

void launch_board_poses_tangent(const PoseProblem& Q, const double4* bear, const int* ok, unsigned char* use, double2* xy_h, int* ok_h, double* q_wc, double* p_wc, double* err, int* valid, cudaStream_t st) {
  if (Q.n_frames <= 0) return;
  board_pose_kernel<double4><<<(Q.n_frames + 3) / 4, 128, 0, st>>>(Q, bear, ok, use, q_wc, p_wc, err, valid, xy_h, ok_h, RsPass{});
  count_launch();
}

// a rolling-shutter refinement-only pass (Q.refine_only = 1) over the views of either residual: meas = double2 normalised points or double4 bearings
template <class M>
static void launch_board_poses_rs(const PoseProblem& Q, const M* meas, const int* ok, unsigned char* use, const RsPass& rsp, double* q_wc, double* p_wc, double* err, int* valid, cudaStream_t st) {
  if (Q.n_frames <= 0) return;
  board_pose_kernel<M, true><<<(Q.n_frames + 3) / 4, 128, 0, st>>>(Q, meas, ok, use, q_wc, p_wc, err, valid, nullptr, nullptr, rsp);
  count_launch();
}

static void launch_view_velocities(int n, const int* order, const double* ts, double max_gap, const double* q_wc, const double* p_wc, const int* valid, double* vel, int* nbr, cudaStream_t st) {
  if (n <= 0) return;
  view_velocity_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, order, ts, max_gap, q_wc, p_wc, valid, vel, nbr);
  count_launch();
}

void launch_board_focal(const PoseProblem& Q, const double2* uv, double cx, double cy, double2* xy, unsigned char* use, double* f2, cudaStream_t st) {
  if (Q.n_frames <= 0) return;
  board_focal_kernel<<<(Q.n_frames + 3) / 4, 128, 0, st>>>(Q, uv, cx, cy, xy, use, f2);
  count_launch();
}

void launch_pinhole_normalize(int n, const double2* uv, double cx, double cy, double f, double2* xy, int* ok, cudaStream_t st) {
  if (n <= 0) return;
  pinhole_normalize_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, uv, cx, cy, 1.0 / f, xy, ok);
  count_launch();
}

static void launch_point_refine(const PointProblem& Q, const double4* bear, double4* board_out, int* optimized, cudaStream_t st, const RsPass* rs) {
  if (Q.n_points <= 0) return;
  const dim3 grid((Q.n_points + 3) / 4);
  if (rs && bear) point_refine_kernel<true, true><<<grid, 128, 0, st>>>(Q, board_out, optimized, bear, *rs);
  else if (rs) point_refine_kernel<false, true><<<grid, 128, 0, st>>>(Q, board_out, optimized, nullptr, *rs);
  else if (bear) point_refine_kernel<true><<<grid, 128, 0, st>>>(Q, board_out, optimized, bear, RsPass{});
  else point_refine_kernel<false><<<grid, 128, 0, st>>>(Q, board_out, optimized, nullptr, RsPass{});
  count_launch();
}

// ---- host drivers of row f1 (icc_pixels_to_normalized, icc_pixels_to_bearings, icc_estimate_board_poses, icc_optimize_board_points,
//      icc_filter_bad_poses) ----
#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status upload_board_views(cudaStream_t st, int np, const double* points, int nf, const int32_t* off, const int32_t* ids, const double* uv, BoardViews& B, std::string& err) {
  const int nc = off[nf];
  B.nf = nf; B.nc = nc; B.np = np;
  CU(B.board.upload(points, np, st)); CU(B.off.upload(off, nf + 1, st)); CU(B.pid.upload(ids, nc, st)); CU(B.uv.upload(uv, nc, st));
  CU(B.xy.alloc(std::max(1, nc))); CU(B.ok.alloc(std::max(1, nc))); CU(B.use.alloc(std::max(1, nc)));
  CU(B.q.alloc(4 * (size_t)nf)); CU(B.p.alloc(3 * (size_t)nf)); CU(B.e.alloc(nf)); CU(B.valid.alloc(nf));
  return ICC_OK;
}

icc_status read_poses(cudaStream_t st, const BoardViews& B, double* q_wc, double* p_wc, double* mean_err, int32_t* valid, std::string& err) {
  CU(cudaMemcpyAsync(q_wc, B.q.p, 4 * (size_t)B.nf * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(p_wc, B.p.p, 3 * (size_t)B.nf * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (mean_err) CU(cudaMemcpyAsync(mean_err, B.e.p, (size_t)B.nf * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(valid, B.valid.p, (size_t)B.nf * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return ICC_OK;
}

icc_status refine_board_points(cudaStream_t st, PointProblem Q, int nc, const int32_t* ids, const std::vector<int>& obs_view, DevBuf<double4>& d_out, std::vector<double>& points_out, int& n_opt, std::string& err,
                               const double4* bear, const RsPass* rs) {
  const int np = Q.n_points;
  std::vector<int> pt_off, pt_obs;
  build_point_adjacency(np, nc, ids, [&](int c) { return obs_view[c] >= 0; }, pt_off, pt_obs);
  DevBuf<int> d_view, d_pt_off, d_pt_obs, d_opt;
  CU(d_view.upload(obs_view)); CU(d_pt_off.upload(pt_off)); CU(d_pt_obs.alloc(std::max<size_t>(1, pt_obs.size()))); CU(d_opt.alloc(np)); CU(d_out.alloc(np));
  if (!pt_obs.empty()) CU(cudaMemcpy(d_pt_obs.p, pt_obs.data(), pt_obs.size() * sizeof(int), cudaMemcpyHostToDevice));
  Q.pt_off = d_pt_off.p; Q.pt_obs = d_pt_obs.p; Q.obs_view = d_view.p;
  launch_point_refine(Q, bear, d_out.p, d_opt.p, st, rs);
  std::vector<int> opt(np); points_out.resize(4 * (size_t)np);
  CU(cudaMemcpyAsync(points_out.data(), d_out.p, (size_t)np * sizeof(double4), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(opt.data(), d_opt.p, (size_t)np * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  n_opt = 0; for (int o : opt) n_opt += o;
  return ICC_OK;
}

// un-projection of every corner and the PoseProblem of EstimatePosesFromJson / OptimizeAllPoses for a W x H camera (pose_estimator.cc:97-101, :181).
// Tangent mode: bearings into B.bear (B.xy and B.okh are the start's scratch); the thresholds keep their values, now on the tangent error.
static PoseProblem unproject_corners(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int W, int H, const BoardViews& B, double max_reproj_error, int min_points, int pose_error) {
  if (pose_error == ICC_POSE_ERROR_TANGENT) launch_bearings(model, intr, B.nc, B.uv.p, B.bear.p, B.ok.p, st);
  else launch_unproject(model, intr, B.nc, B.uv.p, B.xy.p, B.ok.p, st);
  PoseProblem Q; memset(&Q, 0, sizeof Q);
  Q.model = model; for (int i = 0; i < MAX_INTR; ++i) Q.intr[i] = intr[i];
  Q.n_frames = B.nf; Q.n_points = B.np; Q.min_points = min_points > 0 ? min_points : 8;
  Q.board = B.board.p; Q.f_off = B.off.p; Q.pid = B.pid.p;
  const double max_px = max_reproj_error > 0.0 ? max_reproj_error : 0.004 * H;            // pose_estimator.cc:97
  Q.thresh_sq = (W > 0 && H > 0) ? max_px / std::sqrt((double)W * W + (double)H * H) : 1e-3;   // :101 (compared with a SQUARED error by theia's RANSAC)
  Q.max_err = max_px;                                                                       // :181 (pixels against a normalised error, as in the reference)
  return Q;
}

icc_status pixels_to_normalized(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int n, const double* uv, double* xy_out, int32_t* ok, std::string& err) {
  DevBuf<double2> d_uv, d_xy; DevBuf<int> d_ok;
  CU(d_uv.upload(uv, n, st)); CU(d_xy.alloc(n)); CU(d_ok.alloc(n));
  launch_unproject(model, intr, n, d_uv.p, d_xy.p, d_ok.p, st);
  CU(cudaMemcpyAsync(xy_out, d_xy.p, (size_t)n * sizeof(double2), cudaMemcpyDeviceToHost, st));
  if (ok) CU(cudaMemcpyAsync(ok, d_ok.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return ICC_OK;
}

icc_status pixels_to_bearings(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int n, const double* uv, double* xyz_out, int32_t* ok, std::string& err) {
  DevBuf<double2> d_uv; DevBuf<double4> d_b; DevBuf<int> d_ok;
  CU(d_uv.upload(uv, n, st)); CU(d_b.alloc(n)); CU(d_ok.alloc(n));
  launch_bearings(model, intr, n, d_uv.p, d_b.p, d_ok.p, st);
  std::vector<double4> b(n);
  CU(cudaMemcpyAsync(b.data(), d_b.p, (size_t)n * sizeof(double4), cudaMemcpyDeviceToHost, st));
  if (ok) CU(cudaMemcpyAsync(ok, d_ok.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) { xyz_out[3 * i] = b[i].x; xyz_out[3 * i + 1] = b[i].y; xyz_out[3 * i + 2] = b[i].z; }
  return ICC_OK;
}

// the pose kernel of the selected residual on the views of B
static void launch_views(const PoseProblem& Q, BoardViews& B, int pose_error, cudaStream_t st) {
  if (pose_error == ICC_POSE_ERROR_TANGENT) launch_board_poses_tangent(Q, B.bear.p, B.ok.p, B.use.p, B.xy.p, B.okh.p, B.q.p, B.p.p, B.e.p, B.valid.p, st);
  else launch_board_poses(Q, B.xy.p, B.ok.p, B.use.p, B.q.p, B.p.p, B.e.p, B.valid.p, st);
}

static icc_status alloc_tangent(int pose_error, BoardViews& B, std::string& err) {
  if (pose_error == ICC_POSE_ERROR_TANGENT) { CU(B.bear.alloc(std::max(1, B.nc))); CU(B.okh.alloc(std::max(1, B.nc))); }
  return ICC_OK;
}

// Rolling shutter: the views' time order, the largest neighbour gap (2.5 x the median positive spacing of the view times; -1 when there is
// none, so that no view has a neighbour) and the per-view velocities and neighbour counts of the rolling-shutter passes
struct RsState { DevBuf<int> order, nbr; DevBuf<double> ts, vel; double max_gap = -1.0; };

static icc_status rs_prepare(cudaStream_t st, int nf, const double* frame_t, RsState& R, std::string& err) {
  std::vector<int> order(nf);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return frame_t[a] < frame_t[b]; });
  std::vector<double> ts(nf), gaps;
  for (int i = 0; i < nf; ++i) ts[i] = frame_t[order[i]];
  for (int i = 1; i < nf; ++i) if (ts[i] - ts[i - 1] > 0.0) gaps.push_back(ts[i] - ts[i - 1]);
  if (!gaps.empty()) {
    std::sort(gaps.begin(), gaps.end());
    const size_t m = gaps.size() / 2;
    R.max_gap = 2.5 * (gaps.size() % 2 ? gaps[m] : 0.5 * (gaps[m - 1] + gaps[m]));
  }
  CU(R.order.upload(order.data(), nf, st)); CU(R.ts.upload(ts.data(), nf, st)); CU(R.vel.alloc(6 * (size_t)nf)); CU(R.nbr.alloc(nf));
  return ICC_OK;
}

// the velocities of B's views from their current poses
static void rs_velocities(BoardViews& B, RsState& R, cudaStream_t st) {
  launch_view_velocities(B.nf, R.order.p, R.ts.p, R.max_gap, B.q.p, B.p.p, B.valid.p, R.vel.p, R.nbr.p, st);
}

// one rolling-shutter pass (Q.refine_only = 1): the velocities from the current poses, then the refinement of every valid view with them
static void rs_pass(const PoseProblem& Q, BoardViews& B, int pose_error, RsState& R, double line_delay, cudaStream_t st) {
  rs_velocities(B, R, st);
  const RsPass rsp{B.uv.p, R.vel.p, line_delay};
  if (pose_error == ICC_POSE_ERROR_TANGENT) launch_board_poses_rs(Q, B.bear.p, B.ok.p, B.use.p, rsp, B.q.p, B.p.p, B.e.p, B.valid.p, st);
  else launch_board_poses_rs(Q, B.xy.p, B.ok.p, B.use.p, rsp, B.q.p, B.p.p, B.e.p, B.valid.p, st);
}

// the velocities of the last pass and the number of valid views without a neighbour to the caller (both optional); waits for the stream
static icc_status rs_read(cudaStream_t st, int nf, RsState& R, const PoseShutter& S, std::string& err) {
  std::vector<int> nbr(nf);
  if (S.vel) CU(cudaMemcpyAsync(S.vel, R.vel.p, 6 * (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(nbr.data(), R.nbr.p, (size_t)nf * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (S.n_static) *S.n_static = (int32_t)std::count(nbr.begin(), nbr.end(), 0);
  return ICC_OK;
}

icc_status estimate_board_poses(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int W, int H, int np, const double* points, int nf, const int32_t* off,
                                const int32_t* ids, const double* uv, double max_reproj_error, int min_points, int pose_error, const PoseShutter& shutter, double* q_wc, double* p_wc, double* mean_err,
                                int32_t* valid, std::string& err) {
  BoardViews B;
  icc_status rc = upload_board_views(st, np, points, nf, off, ids, uv, B, err); if (rc != ICC_OK) return rc;
  rc = alloc_tangent(pose_error, B, err); if (rc != ICC_OK) return rc;
  PoseProblem Q = unproject_corners(st, model, intr, W, H, B, max_reproj_error, min_points, pose_error);
  launch_views(Q, B, pose_error, st);
  RsState R;
  if (shutter.line_delay > 0.0) {             // two rolling-shutter passes from the global-shutter poses; a view dropped by a pass stays dropped
    rc = rs_prepare(st, nf, shutter.frame_t, R, err); if (rc != ICC_OK) return rc;
    Q.refine_only = 1;
    for (int pass = 0; pass < 2; ++pass) rs_pass(Q, B, pose_error, R, shutter.line_delay, st);
    rc = rs_read(st, nf, R, shutter, err); if (rc != ICC_OK) return rc;
  }
  rc = read_poses(st, B, q_wc, p_wc, mean_err, valid, err); if (rc != ICC_OK) return rc;
  if (cudaGetLastError() != cudaSuccess) { err = "pose kernels failed"; return ICC_ERR_CUDA; }
  return ICC_OK;
}

icc_status optimize_board_points(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int W, int H, int np, const double* points, int nf, const int32_t* off, const int32_t* ids,
                                 const double* uv, double max_reproj_error, int min_points, int min_observations, int pose_error, const PoseShutter& shutter, double* q_wc, double* p_wc,
                                 double* mean_err, int32_t* valid, std::vector<double>& points_out, int32_t* n_opt_out, std::string& err) {
  BoardViews B;
  icc_status rc = upload_board_views(st, np, points, nf, off, ids, uv, B, err); if (rc != ICC_OK) return rc;
  rc = alloc_tangent(pose_error, B, err); if (rc != ICC_OK) return rc;
  const int nc = B.nc;
  const bool rolling = shutter.line_delay > 0.0;
  RsState R;
  if (rolling) { rc = rs_prepare(st, nf, shutter.frame_t, R, err); if (rc != ICC_OK) return rc; }
  CU(B.q.upload(q_wc, 4 * (size_t)nf, st)); CU(B.p.upload(p_wc, 3 * (size_t)nf, st)); CU(B.valid.upload(valid, nf, st));
  CU(cudaMemsetAsync(B.e.p, 0, (size_t)nf * sizeof(double), st));   // views that are not valid keep a zero error
  PoseProblem Q = unproject_corners(st, model, intr, W, H, B, max_reproj_error, min_points, pose_error);
  Q.refine_only = 1;
  // 1. the stored poses and their inlier sets (what the pose dataset holds after EstimatePosesFromJson); rolling shutter: one pass
  if (rolling) rs_pass(Q, B, pose_error, R, shutter.line_delay, st);
  else launch_views(Q, B, pose_error, st);
  std::vector<unsigned char> use(std::max(1, nc)); std::vector<int> vh(nf); std::vector<double> qh(4 * (size_t)nf), ph(3 * (size_t)nf);
  CU(cudaMemcpyAsync(use.data(), B.use.p, (size_t)std::max(1, nc), cudaMemcpyDeviceToHost, st));
  rc = read_poses(st, B, qh.data(), ph.data(), nullptr, vh.data(), err); if (rc != ICC_OK) return rc;
  // 2. OptimizeBoardPoints: one warp per point over its inlier observations in valid views, cameras constant (rolling shutter: with the
  //    velocities of the poses of step 1)
  std::vector<int> obs_view(std::max(1, nc), -1);
  for (int f = 0; f < nf; ++f) if (vh[f]) for (int c = off[f]; c < off[f + 1]; ++c) if (use[c]) obs_view[c] = f;
  for (int f = 0; f < nf; ++f) for (int d = 0; d < 3; ++d) qh[4 * f + d] = -qh[4 * f + d];   // R_cw = conj(q_wc)
  DevBuf<double> d_qcw, d_c; DevBuf<double4> d_board2;
  CU(d_qcw.upload(qh)); CU(d_c.upload(ph));
  PointProblem PQ; memset(&PQ, 0, sizeof PQ);
  PQ.model = model; for (int i = 0; i < MAX_INTR; ++i) PQ.intr[i] = intr[i];
  PQ.normalized = 1; PQ.n_points = np; PQ.min_obs = min_observations > 0 ? min_observations : 30; PQ.huber = 1.345;
  PQ.board_in = B.board.p; PQ.meas = B.xy.p; PQ.q_cw = d_qcw.p; PQ.cam_c = d_c.p;
  int n_opt = 0;
  const RsPass rsp{B.uv.p, R.vel.p, shutter.line_delay};
  if (rolling) rs_velocities(B, R, st);
  rc = refine_board_points(st, PQ, nc, ids, obs_view, d_board2, points_out, n_opt, err, pose_error == ICC_POSE_ERROR_TANGENT ? B.bear.p : nullptr, rolling ? &rsp : nullptr);
  if (rc != ICC_OK) return rc;
  // 3. OptimizeAllPoses on the new points (rolling shutter: one pass)
  Q.board = d_board2.p;
  if (rolling) {
    rs_pass(Q, B, pose_error, R, shutter.line_delay, st);
    rc = rs_read(st, nf, R, shutter, err); if (rc != ICC_OK) return rc;
  } else {
    launch_views(Q, B, pose_error, st);
  }
  rc = read_poses(st, B, q_wc, p_wc, mean_err, valid, err); if (rc != ICC_OK) return rc;
  if (cudaGetLastError() != cudaSuccess) { err = "board point kernels failed"; return ICC_ERR_CUDA; }
  if (n_opt_out) *n_opt_out = n_opt;
  return ICC_OK;
}

void filter_bad_poses(int nv, const double* p_wc, int32_t* valid) {
  std::vector<double> z; for (int i = 0; i < nv; ++i) if (valid[i]) z.push_back(p_wc[3 * i + 2]);
  if (z.empty()) return;
  const double med = median_like_reference(z);
  for (int i = 0; i < nv; ++i) if (valid[i] && std::fabs(p_wc[3 * i + 2] - med) > std::fabs(med)) valid[i] = 0;
}

}  // namespace icc
