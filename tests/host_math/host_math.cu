// Host-side test shim for the PRODUCT's __host__ __device__ math (icc_camera.cuh, icc_device_math.cuh): the very functions the CUDA
// kernels inline, compiled for the CPU by nvcc so that the `-m "not gpu"` suite can check them (finite differences, oracle, known
// answers) without a device.  Test infrastructure only; built by tests/test_host_device_math.py into tests/host_math/_build/.
#include "../../openimucameracalibrator_b200/csrc/icc_camera.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_spline_chain.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_vision_rows.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_imu_rows.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_rotinit_math.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_small_linalg.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_points_math.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_trust_region.cuh"

using namespace icc;

namespace {
template <int N> static int chol_n(const double* A_in, double* b_io) {
  double A[N][N], b[N];
  for (int i = 0; i < N; ++i) { b[i] = b_io[i]; for (int j = 0; j < N; ++j) A[i][j] = A_in[N * i + j]; }
  const bool ok = chol_solve<N>(A, b);
  for (int i = 0; i < N; ++i) b_io[i] = b[i];
  return ok ? 1 : 0;
}
// one factorisation, nrhs right-hand sides (row-major nrhs x N), substituted one after the other
template <int N> static int chol_multi_n(const double* A_in, int nrhs, double* B_io) {
  double A[N][N], b[N];
  for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) A[i][j] = A_in[N * i + j];
  const bool ok = chol_factor<N>(A);
  for (int r = 0; r < nrhs; ++r) {
    for (int i = 0; i < N; ++i) b[i] = B_io[N * r + i];
    chol_substitute<N>(A, b);
    for (int i = 0; i < N; ++i) B_io[N * r + i] = b[i];
  }
  return ok ? 1 : 0;
}
}  // namespace

extern "C" {
// project with both Jacobians: out = [u, v, J(6), Jk(20)], returns ok
int hm_project(int model, const double* k, const double* p, int dispatch_fov, double* out) {
  ProjK pk;
  const Proj a = project_with_k(model, k, v3(p[0], p[1], p[2]), dispatch_fov != 0, &pk);
  const Proj b = project(model, k, v3(p[0], p[1], p[2]), dispatch_fov != 0);
  out[0] = a.u; out[1] = a.v;
  for (int i = 0; i < 6; ++i) out[2 + i] = a.J[i];
  for (int i = 0; i < 20; ++i) out[8 + i] = pk.Jk[i];
  // the two dispatchers must agree bit for bit on value and point Jacobian
  int same = a.ok == b.ok && a.u == b.u && a.v == b.v;
  for (int i = 0; i < 6; ++i) same = same && a.J[i] == b.J[i];
  return (a.ok ? 1 : 0) | (same ? 2 : 0);
}
int hm_num_params(int model) { return camera_num_params(model); }
// theia::Camera::PixelToNormalizedCoordinates / z as the pose kernels compute it (damped Gauss-Newton on the forward model)
int hm_unproject(int model, const double* k, double px, double py, double* xy) { double x = 0.0, y = 0.0; const bool ok = unproject_gn(model, k, px, py, x, y); xy[0] = x; xy[1] = y; return ok ? 1 : 0; }
void hm_so3_exp(const double* w, double* q4out, double* ab) { const ExpOut e = so3_exp_jr(v3(w[0], w[1], w[2])); q4out[0] = e.q.x; q4out[1] = e.q.y; q4out[2] = e.q.z; q4out[3] = e.q.w; ab[0] = e.a; ab[1] = e.b; }
void hm_so3_log(const double* q, double* w) { const V3 r = so3_log(q4(q[0], q[1], q[2], q[3])); w[0] = r.x; w[1] = r.y; w[2] = r.z; }
void hm_so3_jr_inv(const double* w, double* m9) { const M3 J = so3_jr_inv(v3(w[0], w[1], w[2])); for (int i = 0; i < 9; ++i) m9[i] = J.m[i]; }
void hm_qrot(const double* q, const double* p, double* out, double* out_inv) {
  const V3 a = qrot(q4(q[0], q[1], q[2], q[3]), v3(p[0], p[1], p[2])), b = qrot_inv(q4(q[0], q[1], q[2], q[3]), v3(p[0], p[1], p[2]));
  out[0] = a.x; out[1] = a.y; out[2] = a.z; out_inv[0] = b.x; out_inv[1] = b.y; out_inv[2] = b.z;
}
// spline coefficients: out = [lam(5) dlam(5) ddlam(5) | c(6) dc(6) ddc(6) dddc(6) | c3(3) dc3(3)]
void hm_coeffs(double u, double* out) {
  cum_coeffs6(u, out, out + 5); cum_coeffs6_dd(u, out + 10);
  coeffs6(u, out + 15, out + 21, out + 27); coeffs6_ddd(u, out + 33);
  coeffs3(u, out + 39); coeffs3_d(u, out + 42);
}
// The SO(3) spline chain of the residual kernels for one observation: knots (6 x (x,y,z,w)), normalised time u, row covector
// m_theta = d r / d theta (right increment of R_w_i)  ->  q_out = R_w_i(u), rows[18] = d r / d eps_j (right increments of the six knots),
// du = d r / d u through the rotation.  Exactly the code path of vision_kernel / imu_kernel: stage_so3_increment, build_chain, so3_knot_row.
void hm_so3_chain(const double* knots, double u, const double* m_theta, double* q_out, double* rows, double* du) {
  static WarpCtx wc;
  for (int i = 0; i < 6; ++i) wc.q[i] = q4(knots[4 * i], knots[4 * i + 1], knots[4 * i + 2], knots[4 * i + 3]);
  for (int i = 0; i < 5; ++i) stage_so3_increment<true>(&wc, i);
  Chain ch;
  build_chain(&wc, u, ch);
  static double Jt[48 * LDJ];
  *du = so3_knot_row(&wc, ch, v3(m_theta[0], m_theta[1], m_theta[2]), Jt, 0, 1.0);
  for (int c = 0; c < 18; ++c) rows[c] = Jt[c * LDJ];
  q_out[0] = ch.q.x; q_out[1] = ch.q.y; q_out[2] = ch.q.z; q_out[3] = ch.q.w;
}
// Both rows [J | r] of one corner exactly as the persistent vision kernel computes them (icc_vision_rows.cuh): window staging
// (stage_frame_increment), vision_corner_rows (x row direct, y row in the parked layout), vision_yrow_expand.
//   so3 = 6 x (x,y,z,w), r3 = 6 x 3, T_ic = (qx,qy,qz,qw,tx,ty,tz), rows = 2 x 44 (row-major), returns 1 when the projection succeeded
int hm_vision_rows(int model, const double* intr10, int fov, const double* so3, const double* r3, double u_so3, double u_r3, const double* T_ic, double ld,
                   const double* X, double ox, double oy, double* rows) {
  static FrameWin W; VisConst K;
  for (int i = 0; i < 5; ++i) stage_frame_increment(W, i, q4(so3[4 * i], so3[4 * i + 1], so3[4 * i + 2], so3[4 * i + 3]), q4(so3[4 * i + 4], so3[4 * i + 5], so3[4 * i + 6], so3[4 * i + 7]));
  W.q0 = q4(so3[0], so3[1], so3[2], so3[3]); W.u_so3 = u_so3; W.u_r3 = u_r3;
  for (int j = 0; j < 6; ++j) W.p[j] = v3(r3[3 * j], r3[3 * j + 1], r3[3 * j + 2]);
  for (int i = 0; i < 10; ++i) K.intr[i] = intr10[i];
  K.Ric = qmat(q4(T_ic[0], T_ic[1], T_ic[2], T_ic[3])); K.tic = v3(T_ic[4], T_ic[5], T_ic[6]); K.ld = ld; K.model = model; K.fov = fov;
  double yr[YR_N], r0, r1;
  vision_corner_rows<-1>(W, K, v3(X[0], X[1], X[2]), ox, oy, rows, 1, yr, r0, r1);
  vision_yrow_expand(yr, rows + 44, 1);
  return r0 == 1e10 ? 0 : 1;
}
void hm_sincos_small(double x, double* s, double* c) { sincos_small(x, s, c); }
// The three accelerometer rows (3 x 40) and the three gyroscope rows (3 x 24) of one IMU sample exactly as the persistent IMU kernel computes them
// (icc_imu_rows.cuh): imu_accel_rows / imu_gyro_rows, then the parked rows expanded the way accel_part / gyro_part of icc_imu_tmem.cu do.
//   Ma, Mg row-major 3x3; knots as in hm_vision_rows; ba, bg = 3 x 3 bias knots
void hm_imu_rows(const double* so3, const double* r3, const double* ba, const double* bg, double u_so3, double u_r3, double u_ba, double u_bg, const double* Ma, const double* Mg,
                 const double* grav, double w_acc, double w_gyr, double inv_so3_dt, double inv_r3_dt, const double* a_meas, const double* g_meas, double* acc_rows, double* gyr_rows) {
  static ImuWin W; ImuConst K;
  for (int i = 0; i < 5; ++i) stage_frame_increment(W.f, i, q4(so3[4 * i], so3[4 * i + 1], so3[4 * i + 2], so3[4 * i + 3]), q4(so3[4 * i + 4], so3[4 * i + 5], so3[4 * i + 6], so3[4 * i + 7]));
  W.f.q0 = q4(so3[0], so3[1], so3[2], so3[3]);
  for (int j = 0; j < 6; ++j) W.f.p[j] = v3(r3[3 * j], r3[3 * j + 1], r3[3 * j + 2]);
  for (int j = 0; j < 3; ++j) { W.ba[j] = v3(ba[3 * j], ba[3 * j + 1], ba[3 * j + 2]); W.bg[j] = v3(bg[3 * j], bg[3 * j + 1], bg[3 * j + 2]); }
  for (int i = 0; i < 9; ++i) { K.Ma[i] = Ma[i]; K.Mg[i] = Mg[i]; }
  K.grav = v3(grav[0], grav[1], grav[2]); K.w_acc = w_acc; K.w_gyr = w_gyr; K.idt2 = inv_r3_dt * inv_r3_dt; K.inv_so3_dt = inv_so3_dt;
  double pa[ACC_PARK], ra[3];
  imu_accel_rows(W, K, u_so3, u_r3, u_ba, v3(a_meas[0], a_meas[1], a_meas[2]), acc_rows, 1, pa, ra);
  for (int k = 1; k <= 2; ++k) {
    double so3row[18];
    for (int c = 0; c < 18; ++c) so3row[c] = pa[18 * (k - 1) + c];
    imu_accel_row_expand(so3row, q4(pa[36], pa[37], pa[38], pa[39]), pa[39 + k], pa[42], K, k, acc_rows + 40 * k, 1);
  }
  double pg[GYR_PARK], rg[3];
  imu_gyro_rows(W, K, u_so3, u_bg, v3(g_meas[0], g_meas[1], g_meas[2]), gyr_rows, 1, pg, rg);
  for (int k = 1; k <= 2; ++k) {
    for (int c = 0; c < 18; ++c) gyr_rows[24 * k + c] = pg[18 * (k - 1) + c];
    gyr_rows[24 * k + 18] = pg[35 + k];
    for (int c = 19; c < 24; ++c) gyr_rows[24 * k + c] = 0.0;
  }
}
// ---- scalar pieces of the rotation / time-offset initialiser (icc_rotinit_math.cuh) ----------------------------------------------------
int hm_nearest_sorted(const double* ts, int n, double t, double* dist) { double d = 0.0; const int i = nearest_sorted(ts, n, t, d); *dist = d; return i; }
void hm_slerp4(const double* a, const double* b, double t, double* out) {
  const double4 r = slerp4(make_double4(a[0], a[1], a[2], a[3]), make_double4(b[0], b[1], b[2], b[3]), t);
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
void hm_eig4_max(const double* A16, double* q4out) {
  double A[4][4], q[4];
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) A[i][j] = A16[4 * i + j];
  eig4_max(A, q);
  for (int i = 0; i < 4; ++i) q4out[i] = q[i];
}
// ---- small dense linear algebra of the upstream kernels (icc_small_linalg.cuh), at every size they instantiate -------------------------
int hm_chol_solve(int n, const double* A, double* b) {
  switch (n) {
    case 3: return chol_n<3>(A, b); case 6: return chol_n<6>(A, b); case 8: return chol_n<8>(A, b);
    case 10: return chol_n<10>(A, b); case 12: return chol_n<12>(A, b); default: return -1;
  }
}
int hm_chol_factor_substitute(int n, const double* A, int nrhs, double* B) {
  switch (n) {
    case 3: return chol_multi_n<3>(A, nrhs, B); case 6: return chol_multi_n<6>(A, nrhs, B);
    case 8: return chol_multi_n<8>(A, nrhs, B); case 10: return chol_multi_n<10>(A, nrhs, B); case 12: return chol_multi_n<12>(A, nrhs, B);
    default: return -1;
  }
}
void hm_quat_from_columns(const double* R9 /* row-major */, double* q) {
  const Q4 r = quat_from_columns(v3(R9[0], R9[3], R9[6]), v3(R9[1], R9[4], R9[7]), v3(R9[2], R9[5], R9[8]));
  q[0] = r.x; q[1] = r.y; q[2] = r.z; q[3] = r.w;
}
}

// ceres::HomogeneousVectorParameterization(4) of a board point exactly as icc_points.cu uses it (icc_points_math.cuh)
extern "C" void hm_points_prepare(const double* x4, double* board4, double* jac12) { icc::points_prepare(x4, board4, jac12); }
extern "C" void hm_points_plus(const double* x4, const double* d3, double* out4) { icc::points_plus(x4, d3, out4); }

// ---- the trust-region controller of every LM driver (icc_trust_region.cuh), on an opaque buffer of hm_tr_size() bytes ------------------
//   d = function, parameter, gradient tolerance, initial, max, min radius, min relative decrease; i = max iterations, max invalid, check convergence
//   state = radius, decrease factor, cost, initial cost, invalid, iterations, successful, termination, jacobian stale
extern "C" {
int hm_tr_size() { return (int)sizeof(icc::TrustRegion); }
void hm_tr_start(void* t, const double* d, const int* i) {
  icc::TrOptions o = icc::ceres_default_options();
  o.function_tolerance = d[0]; o.parameter_tolerance = d[1]; o.gradient_tolerance = d[2]; o.initial_radius = d[3]; o.max_radius = d[4]; o.min_radius = d[5];
  o.min_relative_decrease = d[6]; o.max_iterations = i[0]; o.max_invalid = i[1]; o.check_convergence = i[2];
  *(icc::TrustRegion*)t = icc::tr_start(o);
}
int hm_tr_continue(void* t) { return icc::tr_continue(*(icc::TrustRegion*)t) ? 1 : 0; }
int hm_tr_jacobian(void* t, double cost, double grad_max) { return icc::tr_jacobian(*(icc::TrustRegion*)t, cost, grad_max) ? 1 : 0; }
int hm_tr_step(void* t, int valid, double model_change, double step_norm, double x_norm) { return icc::tr_step(*(icc::TrustRegion*)t, valid != 0, model_change, step_norm, x_norm) ? 1 : 0; }
int hm_tr_candidate(void* t, double cand_cost) { return icc::tr_candidate(*(icc::TrustRegion*)t, cand_cost) ? 1 : 0; }
void hm_tr_state(const void* t, double* s) {
  const icc::TrustRegion& T = *(const icc::TrustRegion*)t;
  s[0] = T.radius; s[1] = T.decrease_factor; s[2] = T.cost; s[3] = T.initial_cost; s[4] = T.invalid; s[5] = T.iterations; s[6] = T.successful; s[7] = T.termination; s[8] = T.jacobian_stale;
}
}
