// Ceres 2.1 TrustRegionMinimizer step control with the LevenbergMarquardtStrategy radius schedule: the one copy used by every LM
// driver (spline LM and camera calibration in icc_api.cu, static IMU fits in icc_static_imu_math.cuh).  It sees only scalars; each
// driver keeps its loop and may evaluate the candidate before tr_step or only when tr_step asks for it:
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

}  // namespace icc
