// Per-thread pieces of the static multi-pose IMU calibration (icc_static_imu.cu): kept __host__ __device__ in a header so that
// tests/static_imu/static_imu_host_math.cu can compile exactly this code for the CPU.
//
// Reference (imu_tk method of Tedaldi et al., ICRA 2014, as carried by the reference):
//   MultiPosAccResidual / MultiPosGyroResidual          include/OpenCameraCalibrator/core/static_imu_calibrator.h
//   ThreeAxisSensorCalibParams                          include/OpenCameraCalibrator/utils/types.h:170-323
//   QuatIntegrationStepRK4 / IntegrateGyroInterval      include/OpenCameraCalibrator/utils/gyro_integration.h:82-178
//   Ceres 2.1 TrustRegionMinimizer + LevenbergMarquardtStrategy with the default Solver::Options (static_imu_calibrator.cc:120-128,
//   :310-318 only change the linear solver and the progress output).
//
// The gyroscope integration: one RK4 step of the reference is q <- normalize(A_k q) with A_k a 4x4 polynomial in the calibrated
// rates w_k, w_{k+1} and dt.  Normalisation is a positive scale, so the per-step-normalised chain equals normalize(A_{n-1} ... A_0 q0)
// (and so does its derivative).  The kernel evaluates that product as a tree of chunk products; every element is a Dual4x4 =
// (P, dP/dtheta_j) for one parameter direction j, and (P2, D2) o (P1, D1) = (P2 P1, D2 P1 + P2 D1) is plain dual-number matrix
// multiplication.
#pragma once
#include "icc_device_math.cuh"
#include "icc_small_linalg.cuh"
#include "icc_trust_region.cuh"

namespace icc {
namespace simu {

// ---- forward-mode dual number (value, derivative along one direction) ----------------------------------------------------------
struct Dual { double v, d; };
ICC_HD Dual dual(double v, double d = 0.0) { Dual r; r.v = v; r.d = d; return r; }
ICC_HD Dual operator+(Dual a, Dual b) { return dual(a.v + b.v, a.d + b.d); }
ICC_HD Dual operator-(Dual a, Dual b) { return dual(a.v - b.v, a.d - b.d); }
ICC_HD Dual operator-(Dual a) { return dual(-a.v, -a.d); }
ICC_HD Dual operator*(Dual a, Dual b) { return dual(a.v * b.v, a.d * b.v + a.v * b.d); }
ICC_HD Dual operator*(double s, Dual a) { return dual(s * a.v, s * a.d); }
ICC_HD Dual operator/(Dual a, Dual b) { const double iv = 1.0 / b.v; return dual(a.v * iv, (a.d - a.v * iv * b.d) * iv); }
ICC_HD Dual sqrt(Dual a) { const double s = ::sqrt(a.v); return dual(s, a.d / (2.0 * s)); }
ICC_HD double val(double a) { return a; }
ICC_HD double val(Dual a) { return a.v; }
template <class T> ICC_HD T cst(double v) { return T(v); }
template <> ICC_HD Dual cst<Dual>(double v) { return dual(v); }

// ---- accelerometer: g_mag - |T K (a - b)|, T = [[1,-p0,p1],[0,1,-p2],[0,0,1]], K = diag(p3,p4,p5), b = p6..8 -------------------
// Closed-form 1x9 Jacobian row (the reference differentiates the same expression with ceres::Jet).
ICC_HD double acc_residual(const double p[9], const double a[3], double g_mag, double J[9]) {
  const double u0 = a[0] - p[6], u1 = a[1] - p[7], u2 = a[2] - p[8];
  const double v0 = p[3] * u0, v1 = p[4] * u1, v2 = p[5] * u2;
  const double c0 = v0 - p[0] * v1 + p[1] * v2, c1 = v1 - p[2] * v2, c2 = v2;
  const double n = ::sqrt((c0 * c0 + c1 * c1) + c2 * c2);
  if (J) {
    const double e0 = -c0 / n, e1 = -c1 / n, e2 = -c2 / n;   // d r / d c
    J[0] = e0 * -v1;
    J[1] = e0 * v2;
    J[2] = e1 * -v2;
    J[3] = e0 * u0;
    J[4] = e0 * (-p[0] * u1) + e1 * u1;
    J[5] = e0 * (p[1] * u2) + e1 * (-p[2] * u2) + e2 * u2;
    J[6] = -(e0 * p[3]);
    J[7] = -(e0 * (-p[0] * p[4]) + e1 * p[4]);
    J[8] = -(e0 * (p[1] * p[5]) + e1 * (-p[2] * p[5]) + e2 * p[5]);
  }
  return g_mag - n;
}

// ---- gyroscope triad: w = T K (x - b), T = [[1,-p0,p1],[p3,1,-p2],[-p4,p5,1]], K = diag(p6,p7,p8), b = p9..11 (or 0) ------------
template <class T>
ICC_HD void gyro_calibrate(const T p[12], bool with_bias, const double x[3], T w[3]) {
  const T z = cst<T>(0.0);
  const T u0 = cst<T>(x[0]) - (with_bias ? p[9] : z), u1 = cst<T>(x[1]) - (with_bias ? p[10] : z), u2 = cst<T>(x[2]) - (with_bias ? p[11] : z);
  const T k0 = p[6] * u0, k1 = p[7] * u1, k2 = p[8] * u2;
  w[0] = k0 - p[0] * k1 + p[1] * k2;
  w[1] = p[3] * k0 + k1 - p[2] * k2;
  w[2] = -(p[4] * k0) + p[5] * k1 + k2;
}

// 0.5 * ComputeOmegaSkew(w) (gyro_integration.h:33-38), quaternion (w, x, y, z), row-major
template <class T>
ICC_HD void half_skew(const T w[3], T S[16]) {
  const T z = cst<T>(0.0);
  const T a = 0.5 * w[0], b = 0.5 * w[1], c = 0.5 * w[2];
  S[0] = z;  S[1] = -a; S[2] = -b; S[3] = -c;
  S[4] = a;  S[5] = z;  S[6] = c;  S[7] = -b;
  S[8] = b;  S[9] = -c; S[10] = z; S[11] = a;
  S[12] = c; S[13] = b; S[14] = -a; S[15] = z;
}

template <class T>
ICC_HD void mat4_mul(const T A[16], const T B[16], T C[16]) {   // C = A B (C must not alias A or B)
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) C[4 * r + c] = ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) + A[4 * r + 3] * B[12 + c];
}

// One QuatIntegrationStepRK4 (gyro_integration.h:82-108) before its normalisation, as a matrix: q_res = A q.
//   k1 = S0 q, k2 = Sm (q + dt/2 k1), k3 = Sm (q + dt/2 k2), k4 = S1 (q + dt k3), q_res = q + dt (k1/6 + k2/3 + k3/3 + k4/6)
// with S = 0.5 * skew and Sm at the midpoint rate.
template <class T>
ICC_HD void rk4_matrix(const T w0[3], const T w1[3], double dt, T A[16]) {
  T wm[3], S0[16], Sm[16], S1[16], K2[16], K3[16], K4[16], M[16];
  for (int i = 0; i < 3; ++i) wm[i] = 0.5 * (w0[i] + w1[i]);
  half_skew(w0, S0); half_skew(wm, Sm); half_skew(w1, S1);
  const double h2 = 0.5 * dt;
  for (int i = 0; i < 16; ++i) M[i] = ((i % 5) == 0 ? cst<T>(1.0) : cst<T>(0.0)) + h2 * S0[i];        // I + dt/2 S0
  mat4_mul(Sm, M, K2);
  for (int i = 0; i < 16; ++i) M[i] = ((i % 5) == 0 ? cst<T>(1.0) : cst<T>(0.0)) + h2 * K2[i];        // I + dt/2 K2
  mat4_mul(Sm, M, K3);
  for (int i = 0; i < 16; ++i) M[i] = ((i % 5) == 0 ? cst<T>(1.0) : cst<T>(0.0)) + dt * K3[i];        // I + dt K3
  mat4_mul(S1, M, K4);
  const double m1 = 1.0 / 6.0, m2 = 1.0 / 3.0;
  for (int i = 0; i < 16; ++i) A[i] = ((i % 5) == 0 ? cst<T>(1.0) : cst<T>(0.0)) + dt * (((m1 * S0[i] + m2 * K2[i]) + m2 * K3[i]) + m1 * K4[i]);
}

// The reference's vector form of the same step, normalised (used by the tests as the yardstick of rk4_matrix)
ICC_HD void rk4_step_reference(const double q[4], const double w0[3], const double w1[3], double dt, double out[4]) {
  double wm[3], S[16], k1[4], k2[4], k3[4], k4[4], t[4];
  for (int i = 0; i < 3; ++i) wm[i] = 0.5 * (w0[i] + w1[i]);
  auto mv = [](const double M[16], const double x[4], double y[4]) { for (int r = 0; r < 4; ++r) y[r] = M[4 * r] * x[0] + M[4 * r + 1] * x[1] + M[4 * r + 2] * x[2] + M[4 * r + 3] * x[3]; };
  half_skew(w0, S); mv(S, q, k1);
  for (int i = 0; i < 4; ++i) t[i] = q[i] + 0.5 * dt * k1[i];
  half_skew(wm, S); mv(S, t, k2);
  for (int i = 0; i < 4; ++i) t[i] = q[i] + 0.5 * dt * k2[i];
  mv(S, t, k3);
  for (int i = 0; i < 4; ++i) t[i] = q[i] + dt * k3[i];
  half_skew(w1, S); mv(S, t, k4);
  const double m1 = 1.0 / 6.0, m2 = 1.0 / 3.0;
  for (int i = 0; i < 4; ++i) out[i] = q[i] + dt * (m1 * k1[i] + m2 * k2[i] + m2 * k3[i] + m1 * k4[i]);
  const double n = ::sqrt(out[0] * out[0] + out[1] * out[1] + out[2] * out[2] + out[3] * out[3]);
  for (int i = 0; i < 4; ++i) out[i] /= n;
}

// Product P = A_{k1-1} ... A_{k0} over the steps k in [k0, k1) of the unbiased gyroscope samples x (3 per sample); dt from the
// timestamps when gyro_dt <= 0 (IntegrateGyroInterval, gyro_integration.h:150-160).  Rescaled by a positive constant whenever its
// Frobenius norm leaves [1, 4] (a unit-quaternion map has norm 2): the final normalisation removes any positive scale.
template <class T>
ICC_HD void chain_product(const T p[12], bool with_bias, const double* __restrict__ x, const double* __restrict__ t, double gyro_dt,
                          int k0, int k1, T P[16]) {
  for (int i = 0; i < 16; ++i) P[i] = cst<T>((i % 5) == 0 ? 1.0 : 0.0);
  if (k0 >= k1) return;
  T w0[3], w1[3], A[16], N[16];
  gyro_calibrate(p, with_bias, x + 3 * (size_t)k0, w0);
  for (int k = k0; k < k1; ++k) {
    gyro_calibrate(p, with_bias, x + 3 * (size_t)(k + 1), w1);
    const double dt = gyro_dt > 0.0 ? gyro_dt : t[k + 1] - t[k];
    rk4_matrix(w0, w1, dt, A);
    mat4_mul(A, P, N);
    double f = 0.0;
    for (int i = 0; i < 16; ++i) { P[i] = N[i]; f += val(N[i]) * val(N[i]); }
    if (!(f >= 1.0 && f <= 16.0)) { const double s = 2.0 / ::sqrt(f); for (int i = 0; i < 16; ++i) P[i] = s * P[i]; }
    for (int i = 0; i < 3; ++i) w0[i] = w1[i];
  }
}

// Residual of one transition from the product P (q = normalize(P e0), identity start): R(q)^T g0 - g1 with R from
// ceres::QuaternionToRotation (scaled rotation / |q|^2), q = (w, x, y, z).
template <class T>
ICC_HD void transition_residual(const T P[16], const double g0[3], const double g1[3], T r[3]) {
  T q[4] = {P[0], P[4], P[8], P[12]};
  const T n = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
  for (int i = 0; i < 4; ++i) q[i] = q[i] / n;
  const T a = q[0], b = q[1], c = q[2], d = q[3];
  const T aa = a * a, ab = a * b, ac = a * c, ad = a * d, bb = b * b, bc = b * c, bd = b * d, cc = c * c, cd = c * d, dd = d * d;
  const T s = cst<T>(1.0) / (((aa + bb) + cc) + dd);
  T R[9];
  R[0] = s * (aa + bb - cc - dd); R[1] = s * (2.0 * (bc - ad)); R[2] = s * (2.0 * (ac + bd));
  R[3] = s * (2.0 * (ad + bc)); R[4] = s * (aa - bb + cc - dd); R[5] = s * (2.0 * (cd - ab));
  R[6] = s * (2.0 * (bd - ac)); R[7] = s * (2.0 * (ab + cd)); R[8] = s * (aa - bb - cc + dd);
  for (int i = 0; i < 3; ++i) r[i] = ((R[i] * cst<T>(g0[0]) + R[3 + i] * cst<T>(g0[1])) + R[6 + i] * cst<T>(g0[2])) - cst<T>(g1[i]);
}

// ---- Levenberg-Marquardt: the dense step of Ceres' LevenbergMarquardtStrategy under the shared trust-region controller ----------
// Up to 12 unknowns; inactive unknowns (i >= n) stay at zero.  Usage:
//   lm_start(L, options, n, x0, cost, H, g);  while (lm_propose(L)) { evaluate at L.xc -> (c, Hc, gc); lm_consider(L, c, Hc, gc); }
struct LmState {
  TrustRegion T;   // T.cost is the cost at x
  int n;
  double x[12], xc[12], scale[12], H[12][12], g[12];
};

ICC_HD double lm_grad_max(const LmState& L) { double m = 0.0; for (int i = 0; i < L.n; ++i) m = fmax(m, fabs(L.g[i])); return m; }

ICC_HD void lm_start(LmState& L, const TrOptions& o, int n, const double x0[12], double cost, const double H[12][12], const double g[12]) {
  L.T = tr_start(o); L.T.cost = cost;   // handed to tr_jacobian with the gradient by the first lm_propose
  L.n = n;
  for (int i = 0; i < 12; ++i) {
    L.x[i] = i < n ? x0[i] : 0.0; L.xc[i] = L.x[i]; L.g[i] = i < n ? g[i] : 0.0;
    for (int j = 0; j < 12; ++j) L.H[i][j] = (i < n && j < n) ? H[i][j] : 0.0;
    L.scale[i] = i < n ? 1.0 / (1.0 + ::sqrt(L.H[i][i])) : 0.0;     // Jacobi scaling, fixed at the first evaluation
  }
}

// Runs iterations until a candidate L.xc needs its cost (returns true) or the minimiser stops (returns false).
ICC_HD bool lm_propose(LmState& L) {
  const int n = L.n;
  TrustRegion& T = L.T;
  while (tr_continue(T)) {
    // x and its Jacobian came with the evaluation that accepted them (or lm_start's); the gradient test comes after the iteration limit
    if (T.jacobian_stale && !tr_jacobian(T, T.cost, lm_grad_max(L))) break;
    double A[12][12], y[12];
    for (int i = 0; i < 12; ++i) for (int j = 0; j < 12; ++j) A[i][j] = (i < n && j < n) ? L.H[i][j] * L.scale[i] * L.scale[j] : (i == j ? 1.0 : 0.0);
    double Hs_y[12], gs[12];
    for (int i = 0; i < 12; ++i) { gs[i] = i < n ? L.scale[i] * L.g[i] : 0.0; y[i] = -gs[i]; }
    // LM diagonal, clamped; Ceres reuses it after a failed step, which is the same value: H and the scaling have not changed
    double M[12][12];
    for (int i = 0; i < 12; ++i) for (int j = 0; j < 12; ++j) M[i][j] = A[i][j] + ((i == j && i < n) ? fmin(fmax(A[i][i], T.o.min_diagonal), T.o.max_diagonal) / T.radius : 0.0);
    const bool ok = chol_solve<12>(M, y);   // M y = -gs
    double yg = 0.0, yHy = 0.0;
    for (int i = 0; i < n; ++i) { double s = 0.0; for (int j = 0; j < n; ++j) s += A[i][j] * y[j]; Hs_y[i] = s; }
    for (int i = 0; i < n; ++i) { yg += y[i] * gs[i]; yHy += y[i] * Hs_y[i]; }
    double step_sq = 0.0, x_sq = 0.0;
    for (int i = 0; i < n; ++i) { const double dx = y[i] * L.scale[i]; L.xc[i] = L.x[i] + dx; step_sq += dx * dx; x_sq += L.x[i] * L.x[i]; }
    if (tr_step(T, ok, -yg - 0.5 * yHy, ::sqrt(step_sq), ::sqrt(x_sq))) return true;
  }
  return false;
}

ICC_HD void lm_consider(LmState& L, double c, const double H[12][12], const double g[12]) {
  if (!tr_candidate(L.T, c)) return;
  for (int i = 0; i < L.n; ++i) { L.x[i] = L.xc[i]; L.g[i] = g[i]; for (int j = 0; j < L.n; ++j) L.H[i][j] = H[i][j]; }
}

}  // namespace simu
}  // namespace icc
