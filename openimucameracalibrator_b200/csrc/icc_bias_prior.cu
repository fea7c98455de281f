// Random-walk prior on the bias splines (icc_set_bias_random_walk, icc_api.cu): cost, residuals, J^T r and J^T J of the prior rows of
// icc_bias_prior.cuh, added to an evaluation that launch_eval has already written on the same stream.
//
// One CTA does the whole prior: a few hundred knots per sensor, a few thousand rows, so the launch costs more than the arithmetic.
//   * rows: every thread takes rows i, i + blockDim, ... in order, writes them to the residual vector and sums 1/2 r^2; block_sums adds the
//     per-thread sums in a fixed order, and thread 0 adds the total to the cost (the normal equations' cost slot, or the cost of a cost-only
//     evaluation).
//   * normal equations (Jacobian mode, bias knots free): every (knot k, axis a) gathers its J^T r entry and the three J^T J entries
//     (k, k), (k, k+1), (k, k+2) of the pentadiagonal block from the <= 3 segments that touch them, segments in increasing order and
//     nodes in order, and adds each to its one place in the border block of the packed normal equations.
// No atomics: each output location is written by one thread with one fixed sum, so the prior's share is the same on every run.  The
// kernel runs after the evaluation kernels on the same stream, so its read-modify-writes see their finished sums.
#include "icc_bias_prior.cuh"
#include "icc_kernels.h"
#include "icc_reduce.cuh"

namespace icc {
namespace {

constexpr int PRIOR_THREADS = 256;

ICC_D double knot_axis(const double4& k, int a) { return a == 0 ? k.x : a == 1 ? k.y : k.z; }

__global__ void __launch_bounds__(PRIOR_THREADS) bias_prior_kernel(BiasPrior B, DeviceProblem P, DeviceState S, int with_jacobian, double* __restrict__ cost_out,
                                                                 double* __restrict__ res_out) {
  __shared__ double red[PRIOR_THREADS / 32][1];
  double cost = 0.0;
  for (int sensor = 0; sensor < 2; ++sensor) {
    if (!B.on[sensor]) continue;
    const double4* __restrict__ kn = sensor == 0 ? S.ba : S.bg;
    const int n = sensor == 0 ? P.n_ba : P.n_bg;
    const int rows = 3 * BIAS_PRIOR_NODES * (n - 2);
    for (int i = threadIdx.x; i < rows; i += blockDim.x) {   // row i = (segment, node, axis), segment-major
      const int s = i / (3 * BIAS_PRIOR_NODES), g = (i / 3) % BIAS_PRIOR_NODES, a = i % 3;
      const double r = bias_prior_row(knot_axis(kn[s], a), knot_axis(kn[s + 1], a), knot_axis(kn[s + 2], a), g, B.c[sensor][a]);
      if (res_out) res_out[B.res_off[sensor] + i] = r;
      cost += 0.5 * r * r;
    }
    const int* __restrict__ col = sensor == 0 ? P.ba_col : P.bg_col;
    if (!with_jacobian || !col) continue;
    for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) {
      const int k = i / 3, a = i % 3;
      const int ck = col[k];
      if (ck < 0) continue;                                   // this sensor's knots are constant under the flags
      const double c = B.c[sensor][a];
      double gk = 0.0, h[3] = {0.0, 0.0, 0.0};
      for (int s = max(0, k - 2); s <= min(k, n - 3); ++s) {
        for (int g = 0; g < BIAS_PRIOR_NODES; ++g) {
          double w[3]; bias_prior_weights(g, w);
          const double r = bias_prior_row(knot_axis(kn[s], a), knot_axis(kn[s + 1], a), knot_axis(kn[s + 2], a), g, c);
          const double jk = c * w[k - s];
          gk += jk * r;
          for (int o = 0; o <= 2 && k + o <= s + 2; ++o) h[o] += jk * c * w[k + o - s];
        }
      }
      P.ne[P.ne_off_g + ck + a] += gk;
      for (int o = 0; o <= 2 && k + o < n; ++o) {
        const int lo = ck + a, hi = col[k + o] + a;             // bias columns increase with the knot: lo <= hi, both in the border
        P.ne[P.ne_off_C + (int64_t)(hi - P.nk) * P.nb + (lo - P.nk)] += h[o];
      }
    }
  }
  double tot[1]; const double mine[1] = {cost};
  block_sums<1>(mine, red, tot);
  if (threadIdx.x == 0) {
    if (with_jacobian) P.ne[P.ne_off_cost] += tot[0];
    if (cost_out) *cost_out += tot[0];
  }
}

}  // namespace

void launch_bias_prior(const BiasPrior& B, const DeviceProblem& P, const DeviceState& S, bool with_jacobian, double* cost_out, double* residuals_out, cudaStream_t st) {
  if (!B.on[0] && !B.on[1]) return;
  bias_prior_kernel<<<1, PRIOR_THREADS, 0, st>>>(B, P, S, with_jacobian ? 1 : 0, cost_out, residuals_out);
  count_launch();
}

}  // namespace icc
