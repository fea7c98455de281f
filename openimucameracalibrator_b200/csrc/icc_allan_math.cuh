// Per-thread and host pieces of the Allan variance characterisation (icc_allan.cu): kept in a header so that
// tests/allan/allan_host_math.cu can compile exactly this code for the CPU.
//
// Reference (imu_utils by Gao Wenliang, as carried by the reference):
//   AllanGyr / AllanAcc: calcThetas, initStrides, getLogSpace, calcVariance       src/allanvariance/allan_gyr.cc, allan_acc.cc
//   FitAllanGyr / FitAllanAcc: AllanSigmaError, checkData, initValue, getters      src/allanvariance/fitallan_*.cc, include/.../fitallan_*.h
//   AllanVarianceFitter::RunFit                                                    src/core/allan_variance_fitter.cc
#pragma once
#include "icc_device_math.cuh"
#include "icc_trust_region.cuh"

#include <cmath>
#include <vector>

namespace icc {
namespace allan {

constexpr double kLn10 = 2.302585092994045684;

// The curves of the last icc_allan_variance (icc_get_allan_curves): factors and tau are shared by the six channels
struct Curves {
  std::vector<int> factors;
  std::vector<double> tau, sigma2[6], fit_deviation[6];
};

// initStrides + getLogSpace (allan_gyr.cc:137-197), bit for bit: maxStride is the largest power of two <= n/2 (1 when n/2 < 1);
// the log space has float end points and a float exponent 1/(n_clusters-1) and is built by repeated multiplication; every value is
// rounded up and consecutive duplicates are dropped.  The last factor can exceed maxStride by one, and n - 2 factor can then be
// zero or negative: the reference's variance there is 0/0 or -0, and so is ours.
inline std::vector<int> factors(int n, int n_clusters) {
  int mode = n / 2;
  unsigned int max_stride = 1;
  int shft = 0;
  while (mode) { mode = mode >> 1; max_stride = 1u << shft; shft++; }
  const float a = 0.0f, b = (float)std::log10((double)max_stride);
  const double start = std::pow(10.0, (double)a), end = std::pow(10.0, (double)b);
  const double progression = std::pow(end / start, (double)((float)1 / (n_clusters - 1)));
  std::vector<double> ls(n_clusters);
  ls[0] = start;
  for (int i = 1; i < n_clusters; ++i) ls[i] = ls[i - 1] * progression;
  for (double& v : ls) v = std::ceil(v);
  std::vector<int> f(1, (int)ls[0]);
  for (int i = 1; i < n_clusters; ++i) if (ls[i] != ls[i - 1]) f.push_back((int)ls[i]);
  return f;
}

// calcVariance's divisor 2 (period m)^2 (n - 2m), in the reference's order
ICC_HD double variance_divisor(double period, int m, int n) {
  const double cp2 = (period * m) * (period * m);
  return 2 * cp2 * (n - 2 * m);
}

// calcSigma2 (fitallan_gyr.cc:140-149): the five-term Allan variance model
ICC_HD double model(const double p[5], double tau) {
  return p[0] * p[0] / (tau * tau) + p[1] * p[1] / tau + p[2] * p[2] + p[3] * p[3] * tau + p[4] * p[4] * tau * tau;
}

// AllanSigmaError: r = log10(model) - log10(sigma2) with log10(x) = log(x) / log(10); closed-form Jacobian row
ICC_HD double residual(const double p[5], double tau, double log10_sigma2, double J[5]) {
  const double m = model(p, tau);
  if (J) {
    const double s = 1.0 / (m * kLn10);
    J[0] = 2.0 * p[0] / (tau * tau) * s; J[1] = 2.0 * p[1] / tau * s; J[2] = 2.0 * p[2] * s; J[3] = 2.0 * p[3] * tau * s; J[4] = 2.0 * p[4] * tau * tau * s;
  }
  return ::log(m) / kLn10 - log10_sigma2;
}

// FitAllanAcc::checkData (fitallan_acc.cc:119-139): below tau = 1 s a point that raises the running maximum of sigma2 is dropped
inline void accel_filter(const std::vector<double>& sigma2, const std::vector<double>& tau, std::vector<double>& s_out, std::vector<double>& t_out) {
  double run = 0;
  for (size_t i = 0; i < sigma2.size(); ++i) {
    if (tau[i] < 1 && run < sigma2[i]) { run = sigma2[i]; continue; }
    s_out.push_back(sigma2[i]); t_out.push_back(tau[i]);
  }
}

// initValue (fitallan_gyr.cc:66-106): least squares of sqrt(sigma2) on (sqrt tau)^k, k = -2..2, through the inverse of the 5x5
// normal matrix (Eigen's inverse of a dynamic matrix: LU with partial pivoting, then solves against the identity).  `c` is the
// signed solution the reference prints, `init` its absolute value.
inline void init_value(const std::vector<double>& sigma2, const std::vector<double>& tau, double c[5], double init[5]) {
  double A[5][5] = {}, B[5] = {};
  for (size_t i = 0; i < tau.size(); ++i) {
    double F[5];
    for (int k = 0; k < 5; ++k) F[k] = std::pow(std::sqrt(tau[i]), k - 2);
    const double y = std::sqrt(sigma2[i]);
    for (int r = 0; r < 5; ++r) { B[r] += F[r] * y; for (int q = 0; q < 5; ++q) A[r][q] += F[r] * F[q]; }
  }
  int perm[5] = {0, 1, 2, 3, 4};
  for (int k = 0; k < 5; ++k) {   // LU in place, row pivoting on the largest magnitude
    int p = k;
    for (int r = k + 1; r < 5; ++r) if (std::fabs(A[r][k]) > std::fabs(A[p][k])) p = r;
    if (p != k) { for (int q = 0; q < 5; ++q) std::swap(A[k][q], A[p][q]); std::swap(perm[k], perm[p]); }
    if (A[k][k] != 0.0)
      for (int r = k + 1; r < 5; ++r) { A[r][k] /= A[k][k]; for (int q = k + 1; q < 5; ++q) A[r][q] -= A[r][k] * A[k][q]; }
  }
  double inv[5][5];
  for (int col = 0; col < 5; ++col) {
    double y[5];
    for (int r = 0; r < 5; ++r) { double s = perm[r] == col ? 1.0 : 0.0; for (int q = 0; q < r; ++q) s -= A[r][q] * y[q]; y[r] = s; }
    for (int r = 4; r >= 0; --r) { double s = y[r]; for (int q = r + 1; q < 5; ++q) s -= A[r][q] * y[q]; y[r] = s / A[r][r]; }
    for (int r = 0; r < 5; ++r) inv[r][col] = y[r];
  }
  for (int r = 0; r < 5; ++r) { double s = 0.0; for (int q = 0; q < 5; ++q) s += inv[r][q] * B[q]; c[r] = s; init[r] = std::fabs(s); }
}

// Gauss-Newton system of the dogleg: (Hs + mu diag(d^2)) y = bs by Cholesky; false on a non-positive pivot or a non-finite y
// Not chol_solve<5> (icc_small_linalg.cuh), which multiplies by the reciprocal pivot where this divides: the five-parameter fit is so
// ill-conditioned that the last bit of the factor moves a parameter of a run that ends at the iteration limit by up to 1e-4 relative.
ICC_HD bool gn_solve(const double Hs[5][5], const double bs[5], const double d[5], double mu, double y[5]) {
  double L[5][5];
  for (int j = 0; j < 5; ++j) {
    double s = Hs[j][j] + mu * (d[j] * d[j]);
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > 0.0)) return false;
    L[j][j] = ::sqrt(s);
    for (int i = j + 1; i < 5; ++i) { double t = Hs[i][j]; for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k]; L[i][j] = t / L[j][j]; }
  }
  for (int i = 0; i < 5; ++i) { double s = bs[i]; for (int k = 0; k < i; ++k) s -= L[i][k] * y[k]; y[i] = s / L[i][i]; }
  for (int i = 4; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 5; ++k) s -= L[k][i] * y[k]; y[i] = s / L[i][i]; }
  for (int i = 0; i < 5; ++i) if (!(fabs(y[i]) <= 1.7976931348623157e308)) return false;
  return true;
}

// The fit's minimiser state: ceres::Solve with DOGLEG and default options on the point set, from the normal equations of the
// unscaled Jacobian (H = J^T J, b = J^T r) at x.  Usage:
//   fit_start(F, x0, cost, H, b);  while (fit_propose(F)) { evaluate at F.xc -> (c, H, b); fit_consider(F, c, H, b); }
struct Fit {
  Dogleg D;
  double x[5], xc[5], scale[5], H[5][5], b[5];
  double g[5], gn[5], diag[5], alpha;   // dogleg vectors of the current Jacobian (D-scaled space)
  int gn_ok;
};

ICC_HD void fit_start(Fit& F, const double x0[5], double cost, const double H[5][5], const double b[5]) {
  F.D = dl_start(ceres_default_options()); F.D.T.cost = cost;
  if (!(fabs(cost) <= 1.7976931348623157e308)) F.D.T.termination = 4;   // the initial evaluation failed: ceres::Solve stops there
  for (int i = 0; i < 5; ++i) {
    F.x[i] = x0[i]; F.xc[i] = x0[i]; F.b[i] = b[i];
    for (int j = 0; j < 5; ++j) F.H[i][j] = H[i][j];
    F.scale[i] = 1.0 / (1.0 + ::sqrt(H[i][i]));   // Jacobi scaling, fixed at the first evaluation
  }
  F.alpha = 0.0; F.gn_ok = 0;
}

ICC_HD bool fit_propose(Fit& F) {
  TrustRegion& T = F.D.T;
  while (tr_continue(T)) {
    if (T.jacobian_stale) {
      double gmax = 0.0; for (int i = 0; i < 5; ++i) gmax = fmax(gmax, fabs(F.b[i]));
      if (!tr_jacobian(T, T.cost, gmax)) break;
    }
    double Hs[5][5], bs[5];
    for (int i = 0; i < 5; ++i) { bs[i] = F.scale[i] * F.b[i]; for (int j = 0; j < 5; ++j) Hs[i][j] = F.H[i][j] * F.scale[i] * F.scale[j]; }
    if (!F.D.reuse) {
      for (int i = 0; i < 5; ++i) { F.diag[i] = ::sqrt(fmin(fmax(Hs[i][i], T.o.min_diagonal), T.o.max_diagonal)); F.g[i] = bs[i] / F.diag[i]; }
      double gg = 0.0, jg = 0.0, v[5];
      for (int i = 0; i < 5; ++i) { gg += F.g[i] * F.g[i]; v[i] = F.g[i] / F.diag[i]; }
      for (int i = 0; i < 5; ++i) { double s = 0.0; for (int j = 0; j < 5; ++j) s += Hs[i][j] * v[j]; jg += v[i] * s; }
      F.alpha = gg / jg;
      double y[5];
      while (F.D.mu < kDoglegMaxMu && !gn_solve(Hs, bs, F.diag, F.D.mu, y)) F.D.mu *= kDoglegMuIncrease;
      F.gn_ok = F.D.mu < kDoglegMaxMu;
      if (F.gn_ok) for (int i = 0; i < 5; ++i) F.gn[i] = -F.diag[i] * y[i];
    }
    double step[5] = {0, 0, 0, 0, 0}, mc = 0.0, step_sq = 0.0, x_sq = 0.0;
    if (F.gn_ok) {
      F.D.step_norm = dl_dogleg_step<5>(F.g, F.gn, F.diag, F.alpha, T.radius, step);
      double bstep = 0.0, sHs = 0.0;
      for (int i = 0; i < 5; ++i) { double s = 0.0; for (int j = 0; j < 5; ++j) s += Hs[i][j] * step[j]; bstep += bs[i] * step[i]; sHs += step[i] * s; }
      mc = -(bstep + 0.5 * sHs);
    }
    for (int i = 0; i < 5; ++i) { const double dx = step[i] * F.scale[i]; F.xc[i] = F.x[i] + dx; step_sq += dx * dx; x_sq += F.x[i] * F.x[i]; }
    if (dl_step(F.D, F.gn_ok != 0, mc, ::sqrt(step_sq), ::sqrt(x_sq))) return true;
  }
  return false;
}

ICC_HD void fit_consider(Fit& F, double c, const double H[5][5], const double b[5]) {
  if (!dl_candidate(F.D, c)) return;
  for (int i = 0; i < 5; ++i) { F.x[i] = F.xc[i]; F.b[i] = b[i]; for (int j = 0; j < 5; ++j) F.H[i][j] = H[i][j]; }
}

}  // namespace allan
}  // namespace icc
