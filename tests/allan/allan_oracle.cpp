// CPU oracle of the Allan variance characterisation (test infrastructure only): a sequential restatement of
//   AllanGyr / AllanAcc: getAvgDt, calcThetas, initStrides, getLogSpace, calcVariance, getTimes    src/allanvariance/allan_*.cc
//   FitAllanGyr / FitAllanAcc: checkData, initValue, AllanSigmaError under ceres::Solve(DOGLEG)     src/allanvariance/fitallan_*.cc
// The variance is the reference's own loop order.  The fit differentiates the reference's residual with forward-mode Jets (what
// ceres::AutoDiffCostFunction does) and runs Ceres' TrustRegionMinimizer with the traditional dogleg strategy and default options,
// written out here from the documented rules (Jacobi scaling, D = sqrt(clamp(colnorm^2(J))), Cauchy point, regularised Gauss-Newton
// step, radius and mu schedules); residuals and model decreases come from explicit Jacobian rows.  Exported under `icca_` with the
// shapes of include/icc_b200.h, plus the factor set and a fit on given curves.
#include "../../include/icc_b200.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Jet {
  double a, v[5];
  Jet(double x = 0.0) : a(x) { for (double& e : v) e = 0.0; }
};
Jet operator+(const Jet& x, const Jet& y) { Jet r(x.a + y.a); for (int i = 0; i < 5; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
Jet operator-(const Jet& x, const Jet& y) { Jet r(x.a - y.a); for (int i = 0; i < 5; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
Jet operator*(const Jet& x, const Jet& y) { Jet r(x.a * y.a); for (int i = 0; i < 5; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
Jet operator/(const Jet& x, const Jet& y) { const double ib = 1.0 / y.a, q = x.a * ib; Jet r(q); for (int i = 0; i < 5; ++i) r.v[i] = (x.v[i] - q * y.v[i]) * ib; return r; }
Jet log(const Jet& x) { Jet r(std::log(x.a)); for (int i = 0; i < 5; ++i) r.v[i] = x.v[i] / x.a; return r; }

// AllanSigmaError::operator() (fitallan_acc.h)
template <class T>
T sigma_error(const T p[5], double tau, double sigma2) {
  const T t(tau);
  const T m = p[0] * p[0] / (t * t) + p[1] * p[1] / t + p[2] * p[2] + p[3] * p[3] * t + p[4] * p[4] * t * t;
  return log(m) / T(std::log(10)) - T(std::log(sigma2) / std::log(10));
}

double model(const double p[5], double tau) {
  return p[0] * p[0] / (tau * tau) + p[1] * p[1] / tau + p[2] * p[2] + p[3] * p[3] * tau + p[4] * p[4] * tau * tau;
}

std::vector<int> factors(int n, int n_clusters) {   // initStrides + getLogSpace
  int mode = n / 2; unsigned int max_stride = 1; int shft = 0;
  while (mode) { mode = mode >> 1; max_stride = 1 << shft; shft++; }
  const float a = 0, b = (float)log10((double)max_stride);
  const double start = pow(10, a), end = pow(10, b);
  const double progression = pow(end / start, (float)1 / (n_clusters - 1));
  std::vector<double> ls{start};
  for (int i = 1; i < n_clusters; ++i) ls.push_back(ls[i - 1] * progression);
  for (double& v : ls) v = ceil(v);
  std::vector<int> f{(int)ls[0]};
  for (int i = 1; i < n_clusters; ++i) if (ls[i] != ls[i - 1]) f.push_back((int)ls[i]);
  return f;
}

struct FitResult { double x[5], c[5], initial_cost, final_cost; int iterations, successful, termination; };

void init_value(const std::vector<double>& s2, const std::vector<double>& tau, double c[5], double x0[5]) {   // initValue
  double A[5][5] = {}, B[5] = {};
  for (size_t i = 0; i < tau.size(); ++i) {
    double F[5];
    for (int k = 0; k < 5; ++k) F[k] = pow(sqrt(tau[i]), k - 2);
    const double y = sqrt(s2[i]);
    for (int r = 0; r < 5; ++r) { B[r] += F[r] * y; for (int q = 0; q < 5; ++q) A[r][q] += F[r] * F[q]; }
  }
  int perm[5] = {0, 1, 2, 3, 4};   // A.inverse(): partial-pivoting LU, then the identity's columns
  for (int k = 0; k < 5; ++k) {
    int p = k;
    for (int r = k + 1; r < 5; ++r) if (fabs(A[r][k]) > fabs(A[p][k])) p = r;
    if (p != k) { for (int q = 0; q < 5; ++q) std::swap(A[k][q], A[p][q]); std::swap(perm[k], perm[p]); }
    if (A[k][k] != 0.0) for (int r = k + 1; r < 5; ++r) { A[r][k] /= A[k][k]; for (int q = k + 1; q < 5; ++q) A[r][q] -= A[r][k] * A[k][q]; }
  }
  double inv[5][5];
  for (int col = 0; col < 5; ++col) {
    double y[5];
    for (int r = 0; r < 5; ++r) { double s = perm[r] == col ? 1.0 : 0.0; for (int q = 0; q < r; ++q) s -= A[r][q] * y[q]; y[r] = s; }
    for (int r = 4; r >= 0; --r) { double s = y[r]; for (int q = r + 1; q < 5; ++q) s -= A[r][q] * y[q]; y[r] = s / A[r][r]; }
    for (int r = 0; r < 5; ++r) inv[r][col] = y[r];
  }
  for (int r = 0; r < 5; ++r) { double s = 0.0; for (int q = 0; q < 5; ++q) s += inv[r][q] * B[q]; c[r] = s; x0[r] = fabs(s); }
}

// residuals r and Jacobian rows J (npts x 5) at x; returns the cost
double evaluate(const std::vector<double>& s2, const std::vector<double>& tau, const double x[5], std::vector<double>& r, std::vector<double>& J) {
  Jet p[5]; for (int i = 0; i < 5; ++i) { p[i] = Jet(x[i]); p[i].v[i] = 1.0; }
  double c = 0.0;
  for (size_t i = 0; i < tau.size(); ++i) {
    const Jet e = sigma_error(p, tau[i], s2[i]);
    r[i] = e.a; for (int k = 0; k < 5; ++k) J[5 * i + k] = e.v[k];
    c += e.a * e.a;
  }
  return 0.5 * c;
}

bool chol_solve(double M[5][5], const double b[5], double y[5]) {
  double L[5][5] = {};
  for (int j = 0; j < 5; ++j) {
    double s = M[j][j]; for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > 0.0)) return false;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 5; ++i) { double t = M[i][j]; for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k]; L[i][j] = t / L[j][j]; }
  }
  for (int i = 0; i < 5; ++i) { double s = b[i]; for (int k = 0; k < i; ++k) s -= L[i][k] * y[k]; y[i] = s / L[i][i]; }
  for (int i = 4; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 5; ++k) s -= L[k][i] * y[k]; y[i] = s / L[i][i]; }
  for (int i = 0; i < 5; ++i) if (!std::isfinite(y[i])) return false;
  return true;
}

FitResult fit(const std::vector<double>& s2, const std::vector<double>& tau) {
  FitResult R; memset(&R, 0, sizeof R);
  double x[5]; init_value(s2, tau, R.c, x);
  const size_t np = tau.size();
  std::vector<double> r(np), J(5 * np), rc(np), Jc(5 * np);
  double cost = evaluate(s2, tau, x, r, J);
  R.initial_cost = cost;
  R.termination = -1;
  if (!std::isfinite(cost)) R.termination = 4;
  double scale[5];
  for (int k = 0; k < 5; ++k) { double s = 0.0; for (size_t i = 0; i < np; ++i) s += J[5 * i + k] * J[5 * i + k]; scale[k] = 1.0 / (1.0 + sqrt(s)); }
  double radius = 1e4, mu = 1e-8, dl_norm = 0.0;
  bool reuse = false, need_grad_test = true;
  int invalid = 0;
  double g[5], gn[5], D[5], alpha = 0.0; bool gn_ok = false;
  while (R.termination < 0) {
    if (R.iterations >= 50) { R.termination = 0; break; }
    // scaled Jacobian Js = J diag(scale)
    double H[5][5] = {}, b[5] = {}, gmax = 0.0;
    for (size_t i = 0; i < np; ++i)
      for (int a = 0; a < 5; ++a) { b[a] += J[5 * i + a] * scale[a] * r[i]; for (int c = 0; c < 5; ++c) H[a][c] += (J[5 * i + a] * scale[a]) * (J[5 * i + c] * scale[c]); }
    if (need_grad_test) {
      for (int a = 0; a < 5; ++a) { double s = 0.0; for (size_t i = 0; i < np; ++i) s += J[5 * i + a] * r[i]; gmax = std::max(gmax, fabs(s)); }
      need_grad_test = false;
      if (gmax <= 1e-10) { R.termination = 3; break; }
    }
    if (!reuse) {
      for (int a = 0; a < 5; ++a) { D[a] = sqrt(std::min(std::max(H[a][a], 1e-6), 1e32)); g[a] = b[a] / D[a]; }
      double gg = 0.0, jg = 0.0;
      for (size_t i = 0; i < np; ++i) { double s = 0.0; for (int a = 0; a < 5; ++a) s += J[5 * i + a] * scale[a] * (g[a] / D[a]); jg += s * s; }
      for (int a = 0; a < 5; ++a) gg += g[a] * g[a];
      alpha = gg / jg;
      gn_ok = false;
      while (mu < 1.0) {
        double M[5][5], y[5];
        for (int a = 0; a < 5; ++a) for (int c = 0; c < 5; ++c) M[a][c] = H[a][c] + (a == c ? mu * D[a] * D[a] : 0.0);
        if (chol_solve(M, b, y)) { for (int a = 0; a < 5; ++a) gn[a] = -D[a] * y[a]; gn_ok = true; break; }
        mu *= 10.0;
      }
    }
    ++R.iterations;
    double step[5] = {0, 0, 0, 0, 0};
    double mc = 0.0;
    if (gn_ok) {
      double gnorm = 0.0, nnorm = 0.0, gdn = 0.0;
      for (int a = 0; a < 5; ++a) { gnorm += g[a] * g[a]; nnorm += gn[a] * gn[a]; gdn += g[a] * gn[a]; }
      gnorm = sqrt(gnorm); nnorm = sqrt(nnorm);
      if (nnorm <= radius) { for (int a = 0; a < 5; ++a) step[a] = gn[a]; dl_norm = nnorm; }
      else if (gnorm * alpha >= radius) { for (int a = 0; a < 5; ++a) step[a] = -(radius / gnorm) * g[a]; dl_norm = radius; }
      else {
        const double ba = -alpha * gdn, aa = pow(alpha * gnorm, 2.0), bmaa = aa - 2 * ba + pow(nnorm, 2.0), c = ba - aa;
        const double d = sqrt(c * c + bmaa * (pow(radius, 2.0) - aa));
        const double beta = c <= 0 ? (d - c) / bmaa : (radius * radius - aa) / (d + c);
        double s = 0.0;
        for (int a = 0; a < 5; ++a) { step[a] = (-alpha * (1.0 - beta)) * g[a] + beta * gn[a]; s += step[a] * step[a]; }
        dl_norm = sqrt(s);
      }
      for (int a = 0; a < 5; ++a) step[a] /= D[a];
      for (size_t i = 0; i < np; ++i) {   // model_cost_change = -(r . J step + |J step|^2 / 2)
        double js = 0.0; for (int a = 0; a < 5; ++a) js += J[5 * i + a] * scale[a] * step[a];
        mc -= r[i] * js + 0.5 * js * js;
      }
    }
    if (!gn_ok || !(mc > 0.0)) {
      if (++invalid >= 5) { R.termination = 4; break; }
      mu *= 10.0; reuse = false;
      continue;
    }
    invalid = 0;
    double xc[5], dn = 0.0, xn = 0.0;
    for (int a = 0; a < 5; ++a) { const double d = step[a] * scale[a]; xc[a] = x[a] + d; dn += d * d; xn += x[a] * x[a]; }
    if (sqrt(dn) <= 1e-8 * (sqrt(xn) + 1e-8)) { R.termination = 2; break; }
    double cc = evaluate(s2, tau, xc, rc, Jc);
    if (!std::isfinite(cc)) cc = 1.7976931348623157e308;
    if (fabs(cost - cc) <= 1e-6 * cost) { R.termination = 1; break; }
    const double rho = (cost - cc) / mc;
    if (!(rho > 1e-3)) {
      radius *= 0.5; reuse = true;
      if (radius < 1e-32) R.termination = 4;
      continue;
    }
    ++R.successful;
    if (rho < 0.25) radius *= 0.5;
    if (rho > 0.75) radius = std::max(radius, 3.0 * dl_norm);
    if (radius < 1e-32) R.termination = 4;
    mu = std::max(1e-8, 2.0 * mu / 10.0);
    reuse = false; need_grad_test = true;
    for (int a = 0; a < 5; ++a) x[a] = xc[a];
    cost = cc; r.swap(rc); J.swap(Jc);
  }
  for (int a = 0; a < 5; ++a) R.x[a] = x[a];
  R.final_cost = cost;
  return R;
}

void min_deviation(const double p[5], const std::vector<double>& tau, double& dmin, int& imin) {   // findMinNum / findMinIndex
  dmin = 1000.0; imin = 0;
  for (size_t i = 0; i < tau.size(); ++i) {
    const double d = sqrt(model(p, tau[i]));
    imin = dmin < d ? imin : (int)i;
    dmin = dmin < d ? dmin : d;
  }
}

struct Oracle {
  std::string err;
  std::vector<int> factors;
  std::vector<double> tau, sigma2[6], dev[6];
};

// fit of one channel's curve (accelerometer channels drop points as FitAllanAcc::checkData) and its derived quantities
void fit_channel(int c, double freq, const std::vector<double>& s2_all, const std::vector<double>& tau_all, double mean_raw, double* params,
                 icc_allan_noise& z, icc_allan_summary& S) {
  std::vector<double> s2, tau;
  if (c < 3) {
    double run = 0;
    for (size_t i = 0; i < s2_all.size(); ++i) {
      if (tau_all[i] < 1) { if (run < s2_all[i]) { run = s2_all[i]; continue; } }
      s2.push_back(s2_all[i]); tau.push_back(tau_all[i]);
    }
  } else { s2 = s2_all; tau = tau_all; }
  const FitResult R = fit(s2, tau);
  for (int k = 0; k < 5; ++k) { params[k] = R.x[k]; S.init_coeffs[k] = R.c[k]; }
  S.n_fit_points = (int)tau.size(); S.iterations = R.iterations; S.successful_steps = R.successful; S.termination = R.termination;
  S.initial_cost = R.initial_cost; S.final_cost = R.final_cost;
  memset(&z, 0, sizeof z);
  double dmin; int imin; min_deviation(R.x, tau, dmin, imin);
  z.bias_instability_tau = tau.empty() ? 0.0 : tau[imin];
  const double white = sqrt(freq) * sqrt(model(R.x, 1));
  z.mean = mean_raw;
  if (c < 3) { z.bias_instability = dmin; z.white_noise = white; }
  else {
    z.mean = mean_raw / 3600;
    z.bias_b = sqrt(R.x[2] * R.x[2]) / 0.6642824703 / (57.3 * 3600);
    z.bias_instability = dmin / (57.3 * 3600);
    z.white_noise_n = sqrt(freq) * (sqrt(R.x[1] * R.x[1]) / 60.0) * 60 / 57.3;
    z.white_noise = white / (57.3 * 3600);
  }
}

}  // namespace

extern "C" {

icc_status icca_create(void** out, int) { *out = new Oracle(); return ICC_OK; }
void icca_destroy(void* h) { delete static_cast<Oracle*>(h); }
const char* icca_last_error(const void* h) { return static_cast<const Oracle*>(h)->err.c_str(); }
void icca_default_allan_options(icc_allan_options* o) { memset(o, 0, sizeof *o); o->n_clusters = 10000; }

// the factor set (getFactors' first F entries); returns F, writes at most cap
int icca_factors(int n, int n_clusters, int32_t* out, int cap) {
  const std::vector<int> f = factors(n, n_clusters);
  for (int i = 0; i < (int)f.size() && i < cap; ++i) out[i] = f[i];
  return (int)f.size();
}

// calcVariance of one channel's raw values x (already scaled as pushed), sequentially
void icca_variance(int n, const double* t, const double* x, int n_clusters, double* tau, double* sigma2) {
  double sum_dt = 0.0, start_t = t[0]; bool first = true;
  for (int i = 0; i < n; ++i) { if (!first) sum_dt += (t[i] - start_t); start_t = t[i]; first = false; }
  const double dt = sum_dt / (n - 1), freq = 1.0 / dt;
  std::vector<double> th; double sum = 0;
  for (int i = 0; i < n; ++i) { sum += x[i]; th.push_back(sum / freq); }
  const std::vector<int> f = factors(n, n_clusters);
  for (size_t i = 0; i < f.size(); ++i) {
    const int m = f[i];
    const double cp2 = (dt * m) * (dt * m), divided = 2 * cp2 * (n - 2 * m);
    const int max = n - 2 * m;
    double s = 0.0;
    for (int k = 0; k < max; k++) { const double temp = (th[k + 2 * m] - 2 * th[k + m] + th[k]); s += (temp * temp); }
    sigma2[i] = s / divided; tau[i] = dt * m;
  }
}

// the fit of channel c on a given curve (F points), with its derived quantities; mean_raw is getAvgValue()
void icca_fit_channel(int c, double freq, int F, const double* tau, const double* sigma2, double mean_raw, double* params, icc_allan_noise* z, icc_allan_summary* S) {
  memset(S, 0, sizeof *S);
  fit_channel(c, freq, std::vector<double>(sigma2, sigma2 + F), std::vector<double>(tau, tau + F), mean_raw, params, *z, *S);
  S->n_factors = F; S->freq = freq; S->period = 1.0 / freq;
}

icc_status icca_allan_variance(void* hv, int n, const double* t, const double* acc, const double* gyr, const icc_allan_options* opt,
                               double params[30], icc_allan_noise noise[6], icc_allan_summary summary[6]) {
  Oracle& O = *static_cast<Oracle*>(hv);
  const int nc = opt ? opt->n_clusters : 10000;
  if (n < 3 || nc < 2) { O.err = "need n >= 3 and n_clusters >= 2"; return ICC_ERR_INVALID_ARGUMENT; }
  O.factors = factors(n, nc);
  const int F = (int)O.factors.size();
  double sum_dt = 0.0; for (int i = 1; i < n; ++i) sum_dt += t[i] - t[i - 1];
  const double period = sum_dt / (n - 1), freq = 1.0 / period;
  std::vector<double> x(n);
  for (int c = 0; c < 6; ++c) {
    double sum = 0.0;
    for (int i = 0; i < n; ++i) { x[i] = c < 3 ? acc[3 * i + c] : gyr[3 * i + c - 3] * 57.3 * 3600; sum += x[i]; }
    O.tau.assign(F, 0.0); O.sigma2[c].assign(F, 0.0);
    icca_variance(n, t, x.data(), nc, O.tau.data(), O.sigma2[c].data());
    memset(&summary[c], 0, sizeof summary[c]);
    fit_channel(c, freq, O.sigma2[c], O.tau, sum / n, params + 5 * c, noise[c], summary[c]);
    summary[c].n_samples = n; summary[c].n_factors = F; summary[c].freq = freq; summary[c].period = period;
    O.dev[c].resize(F);
    for (int i = 0; i < F; ++i) O.dev[c][i] = sqrt(model(params + 5 * c, O.tau[i]));
  }
  return ICC_OK;
}

icc_status icca_get_allan_curves(const void* hv, int channel, int32_t* factors_out, double* tau, double* sigma2, double* dev, int32_t* len) {
  const Oracle& O = *static_cast<const Oracle*>(hv);
  const int32_t need = (int32_t)O.factors.size();
  if (!factors_out) { *len = need; return ICC_OK; }
  if (*len < need) return ICC_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < need; ++i) { factors_out[i] = O.factors[i]; tau[i] = O.tau[i]; sigma2[i] = O.sigma2[channel][i]; dev[i] = O.dev[channel][i]; }
  *len = need;
  return ICC_OK;
}

}  // extern "C"
