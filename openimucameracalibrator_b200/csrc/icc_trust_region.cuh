// Ceres 2.1 TrustRegionMinimizer step control with the LevenbergMarquardtStrategy radius schedule: the one copy used by every LM
// driver (spline LM in icc_api.cu, camera calibration in icc_camcal.cu, static IMU fits in icc_static_imu_math.cuh).  It sees
// only scalars; each driver keeps its loop and may evaluate the candidate before tr_step or only when tr_step asks for it:
//   TrustRegion T = tr_start(options);
//   while (tr_continue(T)) {
//     if (T.jacobian_stale) { evaluate J at x; if (!tr_jacobian(T, cost, max|g|)) break; }
//     solve with T.radius;  if (tr_step(T, solved, model_change, |step|, |x|) && tr_candidate(T, candidate cost)) x <- candidate;
//   }
#pragma once

namespace icc {

struct TrOptions {
  double function_tolerance, parameter_tolerance, gradient_tolerance, initial_radius, max_radius, min_radius, min_relative_decrease;
  double min_diagonal, max_diagonal;   // LM diagonal clamp, read by the drivers' step computation
  int max_iterations, max_invalid;
  int check_convergence;               // 0: no function / parameter / gradient stop (fixed-count runs); the other stops still apply
};

__host__ __device__ __forceinline__ TrOptions ceres_default_options() {   // ceres::Solver::Options defaults (Ceres 2.1, solver.h)
  TrOptions o;
  o.function_tolerance = 1e-6; o.parameter_tolerance = 1e-8; o.gradient_tolerance = 1e-10; o.initial_radius = 1e4; o.max_radius = 1e16;
  o.min_radius = 1e-32; o.min_relative_decrease = 1e-3; o.min_diagonal = 1e-6; o.max_diagonal = 1e32;
  o.max_iterations = 50; o.max_invalid = 5; o.check_convergence = 1;
  return o;
}

struct TrustRegion {
  TrOptions o;
  double radius, decrease_factor, model_change, cost, initial_cost;   // cost at x; initial_cost at the first Jacobian
  int invalid, iterations, successful;
  int termination;      // -1 while running, else icc_summary.termination (0 max iterations, 1-3 function / parameter / gradient, 4 failure)
  int jacobian_stale;   // x has no Jacobian yet (start, accepted step): the driver evaluates one and calls tr_jacobian
};

__host__ __device__ __forceinline__ TrustRegion tr_start(const TrOptions& o) {
  TrustRegion T;
  T.o = o; T.radius = o.initial_radius; T.decrease_factor = 2.0; T.model_change = 0.0; T.cost = 0.0; T.initial_cost = 0.0;
  T.invalid = 0; T.iterations = 0; T.successful = 0; T.termination = -1; T.jacobian_stale = 1;
  return T;
}

__host__ __device__ __forceinline__ bool tr_continue(TrustRegion& T) {
  if (T.termination < 0 && T.iterations >= T.o.max_iterations) T.termination = 0;
  return T.termination < 0;
}

// A fresh Jacobian at x: the gradient max-norm test (a gradient stop counts no iteration)
__host__ __device__ __forceinline__ bool tr_jacobian(TrustRegion& T, double cost, double grad_max) {
  T.cost = cost; if (T.iterations == 0) T.initial_cost = cost;
  T.jacobian_stale = 0;
  if (T.o.check_convergence && grad_max <= T.o.gradient_tolerance) T.termination = 3;
  return T.termination < 0;
}

__host__ __device__ __forceinline__ void tr_shrink(TrustRegion& T) {   // rejected or invalid step
  T.radius = T.radius / T.decrease_factor; T.decrease_factor *= 2.0;
  if (T.radius < T.o.min_radius) T.termination = 4;
}

// A step without a positive model decrease is invalid; max_invalid in a row stop the run.  A valid step faces the parameter
// tolerance.  True when the candidate cost decides the step (tr_candidate).
__host__ __device__ __forceinline__ bool tr_step(TrustRegion& T, bool valid, double model_change, double step_norm, double x_norm) {
  ++T.iterations;
  if (!valid || !(model_change > 0.0)) {
    if (++T.invalid >= T.o.max_invalid) T.termination = 4; else tr_shrink(T);
    return false;
  }
  T.invalid = 0; T.model_change = model_change;
  if (T.o.check_convergence && step_norm <= T.o.parameter_tolerance * (x_norm + T.o.parameter_tolerance)) { T.termination = 2; return false; }
  return true;
}

// Function tolerance, then accept when rho > min_relative_decrease (radius / max(1/3, 1 - (2 rho - 1)^3), capped) or reject.  A
// non-finite candidate cost counts as the largest double.  True when accepted: x moves to the candidate and needs a Jacobian.
__host__ __device__ __forceinline__ bool tr_candidate(TrustRegion& T, double cand_cost) {
  if (!(fabs(cand_cost) <= 1.7976931348623157e308)) cand_cost = 1.7976931348623157e308;
  const double cost_change = T.cost - cand_cost;
  if (T.o.check_convergence && fabs(cost_change) <= T.o.function_tolerance * T.cost) { T.termination = 1; return false; }
  const double rho = cost_change / T.model_change;
  if (!(rho > T.o.min_relative_decrease)) { tr_shrink(T); return false; }
  ++T.successful; T.cost = cand_cost;
  T.radius = fmin(T.o.max_radius, T.radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rho - 1.0, 3.0)));
  T.decrease_factor = 2.0; T.jacobian_stale = 1;
  return true;
}

// ---- Ceres 2.1 DoglegStrategy (TRADITIONAL_DOGLEG) under the same minimiser ------------------------------------------------------
// A restatement written from the documented behaviour of Ceres 2.1 (dogleg_strategy.cc), not from its source.  The iteration, the
// tolerances and the invalid-step limit are the TrustRegion above; only the radius schedule differs, and the strategy keeps the
// regularisation mu of its Gauss-Newton solve and whether the Gauss-Newton and Cauchy vectors of the current Jacobian can be reused:
//   Dogleg D = dl_start(options);
//   while (tr_continue(D.T)) {
//     if (D.T.jacobian_stale) { evaluate J at x; if (!tr_jacobian(D.T, cost, max|g|)) break; }
//     if (!D.reuse) { diagonal, gradient, Cauchy alpha; while (D.mu < kDoglegMaxMu && !solve with D.mu) D.mu *= kDoglegMuIncrease; }
//     step = dl_dogleg_step(...);  if (dl_step(D, solved, model_change, |step|, |x|) && dl_candidate(D, candidate cost)) x <- candidate;
//   }
struct Dogleg {
  TrustRegion T;       // T.radius is the dogleg radius; T.decrease_factor is unused
  double mu;           // Gauss-Newton regularisation: (J^T J + mu diag(D^2)) y = J^T r
  double step_norm;    // norm of the last dogleg step in the D-scaled space (dl_dogleg_step)
  int reuse;           // the Gauss-Newton and Cauchy vectors belong to the current Jacobian (after a rejected step)
};
constexpr double kDoglegMinMu = 1e-8, kDoglegMaxMu = 1.0, kDoglegMuIncrease = 10.0;

__host__ __device__ __forceinline__ Dogleg dl_start(const TrOptions& o) {
  Dogleg D; D.T = tr_start(o); D.mu = kDoglegMinMu; D.step_norm = 0.0; D.reuse = 0;
  return D;
}

// The traditional dogleg step in the D-scaled space from the scaled gradient g, the scaled Gauss-Newton step gn and the Cauchy
// factor alpha: gn inside the radius; else the gradient step cut at the radius when the Cauchy point lies outside; else the point
// of the segment Cauchy point -> gn on the boundary.  Writes step / D (the Jacobi-scaled coordinates); returns the scaled norm.
template <int N>
__host__ __device__ __forceinline__ double dl_dogleg_step(const double g[N], const double gn[N], const double diag[N], double alpha, double radius,
                                                          double step[N]) {
  double gg = 0.0, nn = 0.0, gb = 0.0;
  for (int i = 0; i < N; ++i) { gg += g[i] * g[i]; nn += gn[i] * gn[i]; gb += g[i] * gn[i]; }
  const double g_norm = sqrt(gg), gn_norm = sqrt(nn);
  if (gn_norm <= radius) {
    for (int i = 0; i < N; ++i) step[i] = gn[i] / diag[i];
    return gn_norm;
  }
  if (g_norm * alpha >= radius) {
    for (int i = 0; i < N; ++i) step[i] = (-(radius / g_norm) * g[i]) / diag[i];
    return radius;
  }
  // a = -alpha g (inside), b = gn (outside): beta in [0, 1] with |a + beta (b - a)| = radius
  const double b_dot_a = -alpha * gb;
  const double a_sq = (alpha * g_norm) * (alpha * g_norm);
  const double bma_sq = (a_sq - 2.0 * b_dot_a) + gn_norm * gn_norm;
  const double c = b_dot_a - a_sq;
  const double d = sqrt(c * c + bma_sq * (radius * radius - a_sq));
  const double beta = c <= 0.0 ? (d - c) / bma_sq : (radius * radius - a_sq) / (d + c);
  double s2 = 0.0;
  for (int i = 0; i < N; ++i) { const double v = (-alpha * (1.0 - beta)) * g[i] + beta * gn[i]; s2 += v * v; step[i] = v / diag[i]; }
  return sqrt(s2);
}

// A step without a solved Gauss-Newton system or without a positive model decrease is invalid: mu x 10 and a fresh solve (the
// radius stays); max_invalid in a row stop the run.  A valid step faces the parameter tolerance.  True when the candidate cost
// decides the step (dl_candidate).
__host__ __device__ __forceinline__ bool dl_step(Dogleg& D, bool valid, double model_change, double step_norm, double x_norm) {
  TrustRegion& T = D.T;
  ++T.iterations;
  if (!valid || !(model_change > 0.0)) {
    if (++T.invalid >= T.o.max_invalid) T.termination = 4;
    else { D.mu *= kDoglegMuIncrease; D.reuse = 0; }
    return false;
  }
  T.invalid = 0; T.model_change = model_change;
  if (T.o.check_convergence && step_norm <= T.o.parameter_tolerance * (x_norm + T.o.parameter_tolerance)) { T.termination = 2; return false; }
  return true;
}

// Function tolerance, then accept when rho > min_relative_decrease or reject.  Rejected: radius / 2, the Gauss-Newton and Cauchy
// vectors are reused.  Accepted: rho < 0.25 halves the radius, rho > 0.75 makes it at least 3 |step|, mu / 5 (not below its
// minimum).  The run stops when the radius falls below min_radius.  True when accepted.
__host__ __device__ __forceinline__ bool dl_candidate(Dogleg& D, double cand_cost) {
  TrustRegion& T = D.T;
  if (!(fabs(cand_cost) <= 1.7976931348623157e308)) cand_cost = 1.7976931348623157e308;
  const double cost_change = T.cost - cand_cost;
  if (T.o.check_convergence && fabs(cost_change) <= T.o.function_tolerance * T.cost) { T.termination = 1; return false; }
  const double rho = cost_change / T.model_change;
  if (!(rho > T.o.min_relative_decrease)) {
    T.radius *= 0.5; D.reuse = 1;
    if (T.radius < T.o.min_radius) T.termination = 4;
    return false;
  }
  ++T.successful; T.cost = cand_cost;
  if (rho < 0.25) T.radius *= 0.5;
  if (rho > 0.75) T.radius = fmax(T.radius, 3.0 * D.step_norm);
  if (T.radius < T.o.min_radius) T.termination = 4;
  D.mu = fmax(kDoglegMinMu, 2.0 * D.mu / kDoglegMuIncrease);
  D.reuse = 0; T.jacobian_stale = 1;
  return true;
}

}  // namespace icc
