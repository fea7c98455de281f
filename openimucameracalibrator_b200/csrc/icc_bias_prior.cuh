// Random-walk prior on the bias splines (icc_set_bias_random_walk): the rows the kernel of icc_bias_prior.cu evaluates, shared with the
// host tests (tests/bias_walk/bias_walk_host_math.cu compiles this header for the CPU).
//
// The bias spline is uniform, of order BIAS_N = 3 and not cumulative: in segment s, with u in [0, 1),
//   b(u) = sum_j B_j(u) b_{s+j},  B = (1/2 (1-u)^2, 1/2 (1 + 2u - 2u^2), 1/2 u^2),   b'(u) = (1/dt) sum_j B'_j(u) b_{s+j},  B' = (-(1-u), 1-2u, u).
// A Wiener-process bias of density q per axis has the negative log-likelihood 1/2 int |b'(t)|^2 / q^2 dt.  b' is linear in u, so the
// 2-point Gauss-Legendre rule on [0, 1] (nodes 1/2 -+ 1/(2 sqrt 3), weights 1/2) is exact: per segment s = 0 .. n-3, node g and axis a,
//   r_{s,g,a} = sqrt(dt / 2) b'_a(u_g) / q_a = c_a sum_j B'_j(u_g) b_{s+j,a},   c_a = 1 / (q_a sqrt(2 dt)),
// and 1/2 sum r^2 is the integral over the n - 2 segments.  The rows are linear in the knots, so their Jacobian is the constant c_a B'_j(u_g).
#pragma once
#include <cmath>

namespace icc {

constexpr int BIAS_PRIOR_NODES = 2;   // Gauss-Legendre nodes per segment

// B'_j(u_g), j = 0..2, at node g of a segment
__host__ __device__ inline void bias_prior_weights(int g, double w[3]) {
  const double u = g == 0 ? 0.21132486540518713 : 0.78867513459481287;   // 1/2 -+ 1/(2 sqrt 3)
  w[0] = -(1.0 - u); w[1] = 1.0 - 2.0 * u; w[2] = u;
}

// r_{s,g,a} from the three knot values b_{s,a}, b_{s+1,a}, b_{s+2,a} of axis a and c_a, written with w_0 = -(w_1 + w_2) (the weights of a
// derivative sum to zero) so that equal knots give exactly 0 and a bias far from zero loses no digits to cancellation
__host__ __device__ inline double bias_prior_row(double b0, double b1, double b2, int g, double c) {
  double w[3]; bias_prior_weights(g, w);
  return c * (w[1] * (b1 - b0) + w[2] * (b2 - b0));
}

// c_a of a sensor from its spacing [s] and density q_a
__host__ __device__ inline double bias_prior_scale(double dt_s, double q) { return 1.0 / (q * sqrt(2.0 * dt_s)); }

}  // namespace icc
