// Host-side test shim for the PRODUCT's bias random-walk rows (icc_bias_prior.cuh): the functions the prior kernel inlines, compiled for the
// CPU by nvcc so that the `-m "not gpu"` suite can check them.  Test infrastructure only; built by tests/bias_walk_support.py.
#include "../../openimucameracalibrator_b200/csrc/icc_bias_prior.cuh"

using namespace icc;

extern "C" {
// every prior row of one sensor (knots: n x 3, per-axis densities q[3]) in the residual order of icc_evaluate; returns the row count
int bw_prior_rows(int n, const double* knots, double dt_s, const double* q, double* out) {
  int row = 0;
  for (int s = 0; s + 2 < n; ++s)
    for (int g = 0; g < BIAS_PRIOR_NODES; ++g)
      for (int a = 0; a < 3; ++a)
        out[row++] = bias_prior_row(knots[3 * s + a], knots[3 * (s + 1) + a], knots[3 * (s + 2) + a], g, bias_prior_scale(dt_s, q[a]));
  return row;
}
}  // extern "C"
