// The host and per-thread math of the Allan variance kernels (icc_allan_math.cuh) and the dogleg step control
// (icc_trust_region.cuh) compiled for the CPU, for tests/test_allan_variance.py.
#include "../../openimucameracalibrator_b200/csrc/icc_allan_math.cuh"

using namespace icc;

extern "C" {
int ah_factors(int n, int n_clusters, int* out, int cap) {
  const std::vector<int> f = allan::factors(n, n_clusters);
  for (int i = 0; i < (int)f.size() && i < cap; ++i) out[i] = f[i];
  return (int)f.size();
}

// Dogleg state as 7 doubles: radius, mu, step_norm, reuse, termination, iterations, successful (+ invalid, cost)
static void pack(const Dogleg& D, double* s) {
  s[0] = D.T.radius; s[1] = D.mu; s[2] = D.step_norm; s[3] = D.reuse; s[4] = D.T.termination; s[5] = D.T.iterations; s[6] = D.T.successful;
  s[7] = D.T.invalid; s[8] = D.T.cost;
}
// Drives dl_step / dl_candidate through a script of k steps: row i = (valid, model_change, step_norm, x_norm, candidate cost,
// dogleg step norm); the state after every step goes to out (9 doubles per step).  Starts from cost0 with ceres_default_options.
void ah_dogleg_script(int k, const double* rows, double cost0, double* out) {
  Dogleg D = dl_start(ceres_default_options());
  tr_jacobian(D.T, cost0, 1.0);
  for (int i = 0; i < k; ++i) {
    const double* r = rows + 6 * i;
    if (tr_continue(D.T)) {
      D.step_norm = r[5];
      if (dl_step(D, r[0] != 0.0, r[1], r[2], r[3]) && dl_candidate(D, r[4]) && D.T.termination < 0) tr_jacobian(D.T, D.T.cost, 1.0);
    }
    pack(D, out + 9 * i);
  }
}
double ah_dogleg_step(const double* g, const double* gn, const double* diag, double alpha, double radius, double* step) {
  return dl_dogleg_step<5>(g, gn, diag, alpha, radius, step);
}
}
