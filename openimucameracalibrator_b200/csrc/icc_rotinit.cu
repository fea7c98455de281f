// IMU-to-camera rotation + time-offset initialiser (sm_90a): the step that produces `gyro_to_cam_calibration.json`, i.e. the
// T_i_c_init rotation and the time offset the hot CLI starts from (SURVEY.md §8(f) row f3).
//
// Replaces what the reference runs serially on the CPU in
//   ImuToCameraRotationEstimator::EstimateCameraImuRotation   src/core/imu_to_camera_rotation_estimator.cc:116-274
//   ImuToCameraRotationEstimator::SolveClosedForm             src/core/imu_to_camera_rotation_estimator.cc:39-114
//   utils::InterpolateQuaternions / InterpolateVector3d / FindClosestTimestamp     src/utils/utils.cc:194-261
// The reference's FindClosestTimestamp is a linear scan per query (O(N^2) per objective evaluation, 40+ evaluations); on the
// sorted, distinct timestamps it is given, bisection + comparison of the two neighbours finds the same index.
//
// Mapping to the machine: every stage is data parallel over the IMU samples (one thread per sample): quaternion interpolation
// to the IMU rate, quaternion finite differences -> visual angular velocity, outlier hold, 15-tap moving averages; one
// evaluation of the alignment objective at a candidate time offset = a grid-wide reduction of 15 sums (means + 3x3
// cross-covariance), a single-thread closed-form rotation (Horn's quaternion method on the 3x3 covariance), and a second
// grid-wide reduction of the robust error.  The golden-section search keeps its state on the device: both candidates of an
// iteration are evaluated by the same launches and a one-thread kernel shrinks the bracket, so the host only enqueues launches
// and reads the result once at the end.
#include "icc_device_math.cuh"
#include "icc_host.h"
#include "icc_reduce.cuh"

#include "icc_rotinit_math.cuh"
#include "icc_small_linalg.cuh"

#include <cmath>

namespace icc {

struct RotInitState {
  double a, b, c, d;          // golden-section bracket and its two interior candidates (time offsets, seconds)
  double sums[2][16];         // per candidate: sum vis (3), sum imu (3), sum imu x vis (9), robust error
  double R[2][9], bias[2][3]; // per candidate closed-form solution (row-major)
  double R_best[9], bias_best[3], error;
  int iterations, done;
};
struct RotInitProblem {
  int n;                      // IMU samples inside the common time window
  const double* t;            // their zero-based timestamps (sorted)
  const double* vis;          // smoothed visual angular velocity at those times (3 per sample)
  const double* imu;          // smoothed gyroscope rates (3 per sample)
  double* vis_shift;          // scratch: 2 x 3n, the shifted + interpolated visual rates of both candidates
  RotInitState* state;
  int estimate_bias;
  double tolerance;
  double bias_in[3];
};

namespace {

constexpr double kHuberK = 1.345, kHuberK2 = kHuberK * kHuberK;   // imu_to_camera_rotation_estimator.cc:36-37

// InterpolateQuaternions (utils.cc:220-240): nearest old sample, slerp towards its successor by dist / (t[n+1] - t[n])
__global__ void interp_quat_kernel(int n_old, const double* __restrict__ t_old, const double4* __restrict__ q_old, int n_new, const double* __restrict__ t_new,
                                   double4* __restrict__ q_new) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_new) return;
  double dist;
  const int k = nearest_sorted(t_old, n_old, t_new[i], dist);
  q_new[i] = k < n_old - 1 ? slerp4(q_old[k], q_old[k + 1], dist / (t_old[k + 1] - t_old[k])) : q_old[k];
}

// visual angular velocity from quaternion finite differences (:178-207); flag = component beyond 2 pi
__global__ void angvel_kernel(int n, const double4* __restrict__ q, double dt_imu, double* __restrict__ w_raw, unsigned char* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = i < n - 1 ? i : n - 2;             // the last difference is duplicated (:188)
  double4 d = make_double4(0, 0, 0, 0);
  if (n >= 2) d = make_double4(q[j + 1].x - q[j].x, q[j + 1].y - q[j].y, q[j + 1].z - q[j].z, q[j + 1].w - q[j].w);
  const double4 qi = q[i];
  const double n2 = qi.x * qi.x + qi.y * qi.y + qi.z * qi.z + qi.w * qi.w;
  const Q4 inv = q4(-qi.x / n2, -qi.y / n2, -qi.z / n2, qi.w / n2);          // Eigen inverse = conjugate / squaredNorm
  const Q4 a = qmul(q4(d.x, d.y, d.z, d.w), inv);
  const double s = -2.0 / dt_imu;
  const double wx = s * a.x, wy = s * a.y, wz = s * a.z;
  w_raw[3 * i] = wx; w_raw[3 * i + 1] = wy; w_raw[3 * i + 2] = wz;
  const double lim = 2.0 * 3.14159265358979323846;
  bad[i] = (fabs(wx) > lim || fabs(wy) > lim || fabs(wz) > lim) ? 1 : 0;
}

// suppress extreme velocities (:196-205): a flagged sample repeats its (already repaired) predecessor, or is zero for i <= 1
__global__ void hold_kernel(int n, const double* __restrict__ w_raw, const unsigned char* __restrict__ bad, double* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int j = i;
  while (bad[j] && j > 1) --j;
  const bool zero = bad[j] != 0;                   // reached i <= 1 still flagged
  w[3 * i] = zero ? 0.0 : w_raw[3 * j]; w[3 * i + 1] = zero ? 0.0 : w_raw[3 * j + 1]; w[3 * i + 2] = zero ? 0.0 : w_raw[3 * j + 2];
}

// SimpleMovingAverage(15) (utils/moving_average.h): mean of the last min(i + 1, 15) samples
__global__ void smooth_kernel(int n, const double* __restrict__ x, double* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k0 = i >= 14 ? i - 14 : 0;
  double s0 = 0, s1 = 0, s2 = 0;
  for (int k = k0; k <= i; ++k) { s0 += x[3 * k]; s1 += x[3 * k + 1]; s2 += x[3 * k + 2]; }
  const double inv = 1.0 / (double)(i - k0 + 1);
  y[3 * i] = s0 * inv; y[3 * i + 1] = s1 * inv; y[3 * i + 2] = s2 * inv;
}

// ---- golden-section state on the device -------------------------------------------------------------------------------------
// sums[c][0..2] = sum vis, [3..5] = sum imu, [6..14] = sum imu_a vis_b (row a, column b), [15] = robust error
ICC_D double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  if (warp == 0) t = warp_sum(lane < nw ? red[lane] : 0.0);
  return t;                                        // valid in warp 0
}

// InterpolateVector3d(time_with_offset, timestamps, angVis) (:47-54, utils.cc:242-261) for sample i at offset td.
// The reference reads one element past the end when the nearest sample is the last one (undefined behaviour); here the last
// sample is returned as is.
ICC_D V3 shifted_vis(const RotInitProblem& Q, int i, double td) {
  const double ti = Q.t[i];
  double dist;
  int lo = 0, hi = Q.n;                            // nearest of (t[j] - td) to t[i]
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (Q.t[mid] - td < ti) lo = mid + 1; else hi = mid; }
  int k;
  if (lo == 0) k = 0;
  else if (lo == Q.n) k = Q.n - 1;
  else k = (fabs(ti - (Q.t[lo - 1] - td)) <= fabs(ti - (Q.t[lo] - td))) ? lo - 1 : lo;
  dist = fabs(ti - (Q.t[k] - td));
  const V3 v0 = v3(Q.vis[3 * k], Q.vis[3 * k + 1], Q.vis[3 * k + 2]);
  if (k + 1 >= Q.n) return v0;
  const double f = dist / ((Q.t[k + 1] - td) - (Q.t[k] - td));
  const V3 v1 = v3(Q.vis[3 * k + 3], Q.vis[3 * k + 4], Q.vis[3 * k + 5]);
  return v3((1.0 - f) * v0.x + f * v1.x, (1.0 - f) * v0.y + f * v1.y, (1.0 - f) * v0.z + f * v1.z);   // lerp3d (utils.cc:214-218)
}

__global__ void __launch_bounds__(256) sums_kernel(RotInitProblem Q) {
  __shared__ double red[8];
  if (Q.state->done) return;
  const int c = blockIdx.y;
  const double td = c == 0 ? Q.state->c : Q.state->d;
  double s[15];
#pragma unroll
  for (int k = 0; k < 15; ++k) s[k] = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Q.n; i += gridDim.x * blockDim.x) {
    const V3 v = shifted_vis(Q, i, td);
    Q.vis_shift[(size_t)c * 3 * Q.n + 3 * i] = v.x; Q.vis_shift[(size_t)c * 3 * Q.n + 3 * i + 1] = v.y; Q.vis_shift[(size_t)c * 3 * Q.n + 3 * i + 2] = v.z;
    const double a0 = Q.imu[3 * i], a1 = Q.imu[3 * i + 1], a2 = Q.imu[3 * i + 2];
    s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += a0; s[4] += a1; s[5] += a2;
    s[6] += a0 * v.x; s[7] += a0 * v.y; s[8] += a0 * v.z; s[9] += a1 * v.x; s[10] += a1 * v.y; s[11] += a1 * v.z; s[12] += a2 * v.x; s[13] += a2 * v.y; s[14] += a2 * v.z;
  }
#pragma unroll
  for (int k = 0; k < 15; ++k) { const double t = block_sum(s[k], red); if (threadIdx.x == 0) atomicAdd(&Q.state->sums[c][k], t); }
}

// closed-form rotation (:56-87): Rs = V C U^T of the SVD of P^T Q  ==  the proper rotation maximising tr(R P^T Q), obtained
// here as the dominant eigenvector of Horn's 4x4 matrix (no SVD needed); bias = mean_vis - Rs mean_imu when enabled
__global__ void solve_kernel(RotInitProblem Q) {
  RotInitState* S = Q.state;
  if (S->done) return;
  const int c = threadIdx.x;
  if (c >= 2) return;
  const double n = (double)Q.n;
  const double* s = S->sums[c];
  const double mv[3] = {s[0] / n, s[1] / n, s[2] / n}, mi[3] = {s[3] / n, s[4] / n, s[5] / n};
  double M[3][3];                                   // M[a][b] = sum (imu_a - mean)(vis_b - mean)
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) M[a][b] = s[6 + 3 * a + b] - n * mi[a] * mv[b];
  double N4[4][4] = {
      {M[0][0] + M[1][1] + M[2][2], M[1][2] - M[2][1], M[2][0] - M[0][2], M[0][1] - M[1][0]},
      {M[1][2] - M[2][1], M[0][0] - M[1][1] - M[2][2], M[0][1] + M[1][0], M[2][0] + M[0][2]},
      {M[2][0] - M[0][2], M[0][1] + M[1][0], -M[0][0] + M[1][1] - M[2][2], M[1][2] + M[2][1]},
      {M[0][1] - M[1][0], M[2][0] + M[0][2], M[1][2] + M[2][1], -M[0][0] - M[1][1] + M[2][2]}};
  double qv[4];
  eig4_max(N4, qv);                                 // (w, x, y, z) of the rotation taking imu to vis
  const Q4 q = qnormalized(q4(qv[1], qv[2], qv[3], qv[0]));
  const M3 R = qmat(q);
  for (int k = 0; k < 9; ++k) S->R[c][k] = R.m[k];
  const V3 rm = mul(R, v3(mi[0], mi[1], mi[2]));
  const bool est = Q.estimate_bias != 0;
  S->bias[c][0] = est ? mv[0] - rm.x : 0.0; S->bias[c][1] = est ? mv[1] - rm.y : 0.0; S->bias[c][2] = est ? mv[2] - rm.z : 0.0;
}

__global__ void __launch_bounds__(256) error_kernel(RotInitProblem Q) {
  __shared__ double red[8];
  const RotInitState* S = Q.state;
  if (S->done) return;
  const int c = blockIdx.y;
  M3 R; for (int k = 0; k < 9; ++k) R.m[k] = S->R[c][k];
  const V3 b = v3(S->bias[c][0], S->bias[c][1], S->bias[c][2]);
  double e = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Q.n; i += gridDim.x * blockDim.x) {
    const double* vs = Q.vis_shift + (size_t)c * 3 * Q.n + 3 * i;
    const V3 D = v3(vs[0], vs[1], vs[2]) - (mul(R, v3(Q.imu[3 * i], Q.imu[3 * i + 1], Q.imu[3 * i + 2])) + b);
    const double err = dot(D, D);
    e += err > kHuberK ? 2.0 * kHuberK * sqrt(err) - kHuberK2 : err;       // (:100-107: the SQUARED norm is compared with k)
  }
  const double t = block_sum(e, red);
  if (threadIdx.x == 0) atomicAdd(&Q.state->sums[c][15], t);
}

// one golden-section step (:232-257)
__global__ void golden_kernel(RotInitProblem Q) {
  RotInitState* S = Q.state;
  if (S->done) return;
  const double fc = S->sums[0][15], fd = S->sums[1][15];
  const int keep = fc < fd ? 0 : 1;
  if (keep == 0) S->b = S->d; else S->a = S->c;
  for (int k = 0; k < 9; ++k) S->R_best[k] = S->R[keep][k];
  if (Q.estimate_bias) for (int k = 0; k < 3; ++k) S->bias_best[k] = S->bias[keep][k];
  S->error = keep == 0 ? fc : fd;
  const double g = (1.0 + sqrt(5.0)) / 2.0;
  S->c = S->b - (S->b - S->a) / g; S->d = S->a + (S->b - S->a) / g;
  S->iterations += 1;
  for (int c = 0; c < 2; ++c) for (int k = 0; k < 16; ++k) S->sums[c][k] = 0.0;
  if (!(fabs(S->c - S->d) > Q.tolerance)) S->done = 1;
}

__global__ void init_state_kernel(RotInitProblem Q, double max_offset) {
  RotInitState* S = Q.state;
  const double g = (1.0 + sqrt(5.0)) / 2.0;
  S->a = -max_offset; S->b = max_offset;
  S->c = S->b - (S->b - S->a) / g; S->d = S->a + (S->b - S->a) / g;
  S->iterations = 0; S->error = 0.0;
  for (int c = 0; c < 2; ++c) { for (int k = 0; k < 16; ++k) S->sums[c][k] = 0.0; for (int k = 0; k < 9; ++k) S->R[c][k] = (k % 4 == 0) ? 1.0 : 0.0; for (int k = 0; k < 3; ++k) S->bias[c][k] = 0.0; }
  for (int k = 0; k < 9; ++k) S->R_best[k] = (k % 4 == 0) ? 1.0 : 0.0;
  for (int k = 0; k < 3; ++k) S->bias_best[k] = Q.bias_in[k];
  S->done = !(fabs(S->c - S->d) > Q.tolerance) ? 1 : 0;
}

}  // namespace

void launch_interp_quat(int n_old, const double* t_old, const double4* q_old, int n_new, const double* t_new, double4* q_new, cudaStream_t st) {
  if (n_new <= 0) return;
  interp_quat_kernel<<<(n_new + 255) / 256, 256, 0, st>>>(n_old, t_old, q_old, n_new, t_new, q_new); count_launch();
}

void launch_visual_angular_velocity(int n, const double4* q, double dt_imu, double* w_raw, unsigned char* bad, double* w_held, double* w_smooth, const double* imu, double* imu_smooth, cudaStream_t st) {
  if (n <= 0) return;
  const int g = (n + 255) / 256;
  angvel_kernel<<<g, 256, 0, st>>>(n, q, dt_imu, w_raw, bad); count_launch();
  hold_kernel<<<g, 256, 0, st>>>(n, w_raw, bad, w_held); count_launch();
  smooth_kernel<<<g, 256, 0, st>>>(n, w_held, w_smooth); count_launch();
  smooth_kernel<<<g, 256, 0, st>>>(n, imu, imu_smooth); count_launch();
}

void launch_golden_section(const RotInitProblem& Q, double max_offset, int max_iterations, int sm_count, cudaStream_t st) {
  init_state_kernel<<<1, 1, 0, st>>>(Q, max_offset); count_launch();
  int gx = (Q.n + 255) / 256; if (gx > 4 * sm_count) gx = 4 * sm_count; if (gx < 1) gx = 1;
  for (int it = 0; it < max_iterations; ++it) {
    sums_kernel<<<dim3(gx, 2), 256, 0, st>>>(Q); count_launch();
    solve_kernel<<<1, 32, 0, st>>>(Q); count_launch();
    error_kernel<<<dim3(gx, 2), 256, 0, st>>>(Q); count_launch();
    golden_kernel<<<1, 1, 0, st>>>(Q); count_launch();
  }
}

// ---- host driver of row f3 (icc_estimate_imu_to_camera_rotation) ----------------------------------------------------------
#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status estimate_imu_to_camera_rotation(cudaStream_t st, int sm_count, int n_views, const double* view_t, const double* q_cw, int n_imu, const double* imu_t,
                                           const double* gyro, const double* bias_in, double* q_out, double* td_out, double* bias_out, double* err_out,
                                           int32_t* iters_out, std::string& err) {
  // ---- host preparation (app :96-162): ordered maps, median frame interval, regular grid, common window ------------------
  // std::map semantics of the reference (time ordered, a repeated timestamp keeps the LAST sample); already-sorted input -- the
  // normal case -- skips the tree
  auto ordered = [](const double* t, int n) { std::vector<std::pair<double, int>> o; o.reserve(n);
    bool inc = true; for (int i = 1; i < n && inc; ++i) inc = t[i] > t[i - 1];
    if (inc) { for (int i = 0; i < n; ++i) o.emplace_back(t[i], i); return o; }
    std::map<double, int> m; for (int i = 0; i < n; ++i) m[t[i]] = i;
    for (const auto& kv : m) o.emplace_back(kv.first, kv.second);
    return o; };
  const std::vector<std::pair<double, int>> vmap = ordered(view_t, n_views), gmap = ordered(imu_t, n_imu);
  if (vmap.size() < 2 || gmap.size() < 2) { err = "need at least two distinct view and gyroscope timestamps"; return ICC_ERR_INVALID_ARGUMENT; }
  double imu_dt = 0.0;
  for (int i = 1; i < n_imu; ++i) imu_dt += imu_t[i] - imu_t[i - 1];                     // app :103-108 (file order)
  imu_dt /= (double)(n_imu - 1);
  std::vector<double> tv; std::vector<double4> qv;
  for (const auto& kv : vmap) { tv.push_back(kv.first); const double* q = q_cw + 4 * (size_t)kv.second; qv.push_back(make_double4(q[0], q[1], q[2], q[3])); }
  std::vector<double> diffs; for (size_t i = 1; i < tv.size(); ++i) diffs.push_back(tv[i] - tv[i - 1]);
  const double cam_dt = median_like_reference(diffs);
  if (!(cam_dt > 0.0)) { err = "non-positive median frame interval"; return ICC_ERR_INVALID_ARGUMENT; }
  std::vector<double> grid; for (double t = tv.front(); t < tv.back(); t += cam_dt) grid.push_back(t);   // app :139-144
  std::vector<double> tg, gg;    // gyroscope, time ordered, bias removed
  for (const auto& kv : gmap) { tg.push_back(kv.first); for (int d = 0; d < 3; ++d) gg.push_back(gyro[3 * (size_t)kv.second + d] - (bias_in ? bias_in[d] : 0.0)); }
  const double t0 = grid.front() >= tg.front() ? grid.front() : tg.front();               // :127-129
  const double tend = grid.back() >= tg.back() ? grid.back() : tg.back();                 // (the LATER end, as in the reference)
  std::vector<double> tI, wI; for (size_t i = 0; i < tg.size(); ++i) if (tg[i] >= t0 && tg[i] <= tend) { tI.push_back(tg[i] - t0); for (int d = 0; d < 3; ++d) wI.push_back(gg[3 * i + d]); }
  size_t g0 = 0; while (g0 < grid.size() && grid[g0] < t0) ++g0;
  std::vector<double> tV; for (size_t i = g0; i < grid.size(); ++i) if (grid[i] <= tend) tV.push_back(grid[i] - t0);
  const int N = (int)tI.size(), Mc = (int)tV.size(), M = (int)grid.size(), nv = (int)tv.size();
  if (N < 2 || Mc < 1) { err = "camera and gyroscope streams do not overlap"; return ICC_ERR_INVALID_ARGUMENT; }
  // ---- device pipeline --------------------------------------------------------------------------------------------------
  DevBuf<double> d_tv, d_grid, d_tV, d_tI, d_wI, d_wraw, d_wheld, d_wvis, d_wimu, d_shift; DevBuf<double4> d_qv, d_qgrid, d_qi; DevBuf<unsigned char> d_bad; DevBuf<RotInitState> d_state;
  CU(d_tv.upload(tv)); CU(d_qv.upload(qv)); CU(d_grid.upload(grid)); CU(d_tV.upload(tV)); CU(d_tI.upload(tI)); CU(d_wI.upload(wI));
  CU(d_qgrid.alloc(M)); CU(d_qi.alloc(N)); CU(d_wraw.alloc(3 * (size_t)N)); CU(d_wheld.alloc(3 * (size_t)N)); CU(d_wvis.alloc(3 * (size_t)N)); CU(d_wimu.alloc(3 * (size_t)N));
  CU(d_shift.alloc(6 * (size_t)N)); CU(d_bad.alloc(N)); CU(d_state.alloc(1));
  launch_interp_quat(nv, d_tv.p, d_qv.p, M, d_grid.p, d_qgrid.p, st);              // views -> regular frame grid (app :150-156)
  launch_interp_quat(Mc, d_tV.p, d_qgrid.p + g0, N, d_tI.p, d_qi.p, st);           // grid -> IMU rate (:172-173)
  launch_visual_angular_velocity(N, d_qi.p, imu_dt, d_wraw.p, d_bad.p, d_wheld.p, d_wvis.p, d_wI.p, d_wimu.p, st);
  RotInitProblem Q; memset(&Q, 0, sizeof Q);
  Q.n = N; Q.t = d_tI.p; Q.vis = d_wvis.p; Q.imu = d_wimu.p; Q.vis_shift = d_shift.p; Q.state = d_state.p;
  Q.estimate_bias = bias_in ? 0 : 1; Q.tolerance = 1e-4;
  for (int d = 0; d < 3; ++d) Q.bias_in[d] = bias_in ? bias_in[d] : 0.0;
  // the bracket shrinks by the golden ratio per step whatever the data says, so the step count is known up to rounding
  int n_it = 0; { const double g = (1.0 + std::sqrt(5.0)) / 2.0; double a = -1.0, b = 1.0, c = b - (b - a) / g, d = a + (b - a) / g; while (std::fabs(c - d) > Q.tolerance && n_it < 200) { b = d; c = b - (b - a) / g; d = a + (b - a) / g; ++n_it; } }
  launch_golden_section(Q, 1.0, n_it + 2, sm_count > 0 ? sm_count : 132, st);
  RotInitState S;
  CU(cudaMemcpyAsync(&S, d_state.p, sizeof S, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (cudaGetLastError() != cudaSuccess) { err = "rotation initialiser kernels failed"; return ICC_ERR_CUDA; }
  if (!S.done) { err = "golden-section search did not terminate"; return ICC_ERR_NUMERIC; }
  const double* R = S.R_best;                                                              // row-major
  const Q4 q = quat_from_columns(v3(R[0], R[3], R[6]), v3(R[1], R[4], R[7]), v3(R[2], R[5], R[8]));
  q_out[0] = q.x; q_out[1] = q.y; q_out[2] = q.z; q_out[3] = q.w;
  *td_out = (S.b + S.a) / 2;                                                               // :259
  if (bias_out) for (int d = 0; d < 3; ++d) bias_out[d] = S.bias_best[d];
  if (err_out) *err_out = S.error;
  if (iters_out) *iters_out = S.iterations;
  return ICC_OK;
}

}  // namespace icc
