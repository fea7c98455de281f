// Oracle of the bias-spline spacing and the random-walk prior on the bias splines (icc_set_bias_splines, icc_set_bias_random_walk,
// icc_num_bias_prior_residuals), for tests/test_bias_random_walk.py and tests/test_gpu_bias_random_walk.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more through tests/omni_radtan/omni_oracle.cpp with -DOMNI_TANGENT (every
// camera model and the tangent reprojection error, icco_set_tangent_bearings), with two substitutions made by function-like macros that paste
// the first argument's first token, `o` at every call and `Oracle` at the definition, and so tell the two apart:
//   * every call `evaluate(o, ...)` resolves to evaluate_with_prior below, and the definition is renamed evaluate_oracle;
//   * every call `total_residuals(o)` resolves to total_with_prior, the definition is renamed total_residuals_oracle.
// So the oracle's LM, icco_evaluate, icco_normal_matvec and icco_jacobian_dense all see the prior rows.  They are stated here on their own:
//   * the spline of sensor s over its n knots has n - 2 segments; in segment j, node g (u_g = 1/2 -+ 1/(2 sqrt 3)) and axis a,
//     r = sqrt(dt / 2) b'_a(u_g) / q_a with b'(u) = (1/dt) (-(1-u) b_j + (1-2u) b_{j+1} + u b_{j+2});
//   * rows follow the gyroscope rows: accelerometer prior, then gyroscope prior, segment-major, then node, then axis; only shard 0 has them;
//   * their columns are the bias-knot columns when the flags free them.
// icco_batch_init_spline runs the oracle's own assembly and then, for a spacing other than the reference's 10 s, sizes the bias splines
// again (duration / dt + 3 knots at the start value) and points every IMU block at the knots and the u of its sample time (CalcTimes).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <vector>

namespace { struct Oracle; struct Normal; }
#define evaluate(first, ...) BW_EVAL_##first, __VA_ARGS__)
#define BW_EVAL_o evaluate_with_prior(o
#define BW_EVAL_Oracle evaluate_oracle(Oracle
#define total_residuals(first) BW_TOTAL_##first)
#define BW_TOTAL_o total_with_prior(o
#define BW_TOTAL_const total_residuals_oracle(const
#define icco_batch_init_spline(...) icco_batch_init_spline_base(__VA_ARGS__)
#define icco_create(...) icco_create_base(__VA_ARGS__)
namespace {
void evaluate_with_prior(Oracle& o, double* cost_out, double* residuals, Normal* ne, std::vector<double>* Jdense, int n_res_total);
int total_with_prior(const Oracle& o);
}  // namespace
#define OMNI_TANGENT
#include "../omni_radtan/omni_oracle.cpp"
#undef evaluate
#undef total_residuals
#undef icco_batch_init_spline
#undef icco_create

namespace {

struct Walk {
  double dt_set[2] = {0.0, 0.0};                     // icco_set_bias_splines (<= 0: 10 s)
  bool on_set[2] = {false, false}; double q_set[2][3] = {{0.0}};
  bool on[2] = {false, false}; double q[2][3] = {{0.0}};   // as of the last batch_init
};
std::map<const Oracle*, Walk> g_walk;

int prior_rows(const Oracle& o, int s) {
  const auto it = g_walk.find(&o);
  if (it == g_walk.end() || !it->second.on[s] || o.shard_rank != 0) return 0;
  return 6 * (nknots(s == 0 ? o.ba : o.bg, 3) - 2);
}
int total_with_prior(const Oracle& o) { return total_residuals_oracle(o) + prior_rows(o, 0) + prior_rows(o, 1); }

void evaluate_with_prior(Oracle& o, double* cost_out, double* residuals, Normal* ne, std::vector<double>* Jdense, int n_res_total) {
  double cost = 0.0;
  evaluate_oracle(o, &cost, residuals, ne, Jdense, n_res_total);
  const auto it = g_walk.find(&o);
  int row = total_residuals_oracle(o);
  double prior = 0.0;
  for (int s = 0; s < 2 && it != g_walk.end(); ++s) {
    if (prior_rows(o, s) == 0) continue;
    const std::vector<double>& kn = s == 0 ? o.ba : o.bg;
    const int n = nknots(kn, 3), off = s == 0 ? o.off_ba : o.off_bg;
    const double dt = double(s == 0 ? o.dt_ba_ns : o.dt_bg_ns) * 1e-9;
    for (int j = 0; j + 2 < n; ++j)
      for (int g = 0; g < 2; ++g) {
        const double u = 0.5 + (g == 0 ? -0.5 : 0.5) / std::sqrt(3.0);
        const double dB[3] = {-(1.0 - u), 1.0 - 2.0 * u, u};
        for (int a = 0; a < 3; ++a, ++row) {
          const double f = std::sqrt(dt / 2.0) / (dt * it->second.q[s][a]);
          double r = 0.0; for (int i = 0; i < 3; ++i) r += f * dB[i] * kn[3 * (j + i) + a];
          prior += 0.5 * r * r;
          if (residuals) residuals[row] = r;
          if (off < 0) continue;                           // knots constant under the flags: cost and residuals only
          for (int i = 0; i < 3; ++i) {
            const int ci = off + 3 * (j + i) + a;
            if (Jdense) (*Jdense)[size_t(row) * o.n_tan + ci] = f * dB[i];
            if (!ne) continue;
            ne->g[o.perm[ci]] += f * dB[i] * r;
            for (int k = i; k < 3; ++k) ne->add(o.perm[ci], o.perm[off + 3 * (j + k) + a], f * dB[i] * f * dB[k]);
          }
        }
      }
  }
  cost += prior;
  if (ne) ne->cost = cost;
  if (cost_out) *cost_out = cost;
}

// bias splines at spacing dt (ns) for sensor s: knots at the start value, IMU blocks re-pointed
void respace(Oracle& o, int s, int64_t dt_ns) {
  const int64_t duration = o.end_ns - o.start_ns;
  const int n = int(duration / dt_ns) + BIAS_N;
  std::vector<double>& kn = s == 0 ? o.ba : o.bg;
  const double* b0 = s == 0 ? o.ip.acc_bias : o.ip.gyr_bias;
  kn.assign(3 * size_t(n), 0.0);
  for (int i = 0; i < n; ++i) for (int d = 0; d < 3; ++d) kn[3 * i + d] = b0[d];
  if (s == 0) { o.dt_ba_ns = dt_ns; o.inv_ba_dt = 1.0 / double(dt_ns); } else { o.dt_bg_ns = dt_ns; o.inv_bg_dt = 1.0 / double(dt_ns); }
  for (auto& b : o.blocks) {
    if (b.type != (s == 0 ? BLK_ACCEL : BLK_GYRO)) continue;
    const int64_t t_ns = int64_t(o.imu_used[b.frame].t_s * S_TO_NS);
    double u = 0.0; int64_t seg = 0;
    if (!calc_times(t_ns, o.start_ns, dt_ns, size_t(n), BIAS_N, u, seg)) { fprintf(stderr, "bias_walk_oracle: sample outside the bias spline\n"); abort(); }
    b.u_bias = u;
    const int first = s == 0 ? 2 * SPLINE_N : SPLINE_N;
    for (int i = 0; i < BIAS_N; ++i) b.params[first + i].ptr = &kn[3 * size_t(seg + i)];
  }
  o.cur_flags = -1;
}

}  // namespace

extern "C" {

// a new oracle may reuse a freed one's address: it starts without spacing or prior
icc_status icco_create(void** out, int n_threads) {
  const icc_status st = icco_create_base(out, n_threads);
  if (st == ICC_OK) g_walk.erase(O(*out));
  return st;
}

icc_status icco_set_bias_splines(void* h, double acc_dt_s, double gyr_dt_s) {
  Oracle& o = *O(h);
  for (const double dt : {acc_dt_s, gyr_dt_s})
    if (!std::isfinite(dt) || (dt > 0.0 && (dt * 1e9 < 1.0 || dt > 1e9))) { o.err = "bad bias knot spacing"; return ICC_ERR_INVALID_ARGUMENT; }
  Walk& W = g_walk[&o]; W.dt_set[0] = acc_dt_s; W.dt_set[1] = gyr_dt_s;
  return ICC_OK;
}
icc_status icco_set_bias_random_walk(void* h, const double* acc_q, const double* gyr_q) {
  Oracle& o = *O(h);
  const double* q[2] = {acc_q, gyr_q};
  for (int s = 0; s < 2; ++s) if (q[s]) for (int a = 0; a < 3; ++a) if (!(q[s][a] > 0.0) || !std::isfinite(q[s][a])) { o.err = "bad random-walk density"; return ICC_ERR_INVALID_ARGUMENT; }
  Walk& W = g_walk[&o];
  for (int s = 0; s < 2; ++s) { W.on_set[s] = q[s] != nullptr; for (int a = 0; a < 3; ++a) W.q_set[s][a] = q[s] ? q[s][a] : 0.0; }
  return ICC_OK;
}
icc_status icco_num_bias_prior_residuals(const void* h, int* n) { const Oracle& o = *O(h); *n = prior_rows(o, 0) + prior_rows(o, 1); return ICC_OK; }

icc_status icco_batch_init_spline(void* h, const icc_init_params* ipp) {
  const icc_status st = icco_batch_init_spline_base(h, ipp);
  if (st != ICC_OK) return st;
  Oracle& o = *O(h);
  Walk& W = g_walk[&o];
  for (int s = 0; s < 2; ++s) {
    W.on[s] = W.on_set[s]; for (int a = 0; a < 3; ++a) W.q[s][a] = W.q_set[s][a];
    if (W.dt_set[s] > 0.0 && int64_t(W.dt_set[s] * 1e9) != int64_t(10 * 1e9)) respace(o, s, int64_t(W.dt_set[s] * 1e9));
  }
  return ICC_OK;
}

// per used IMU sample (icco_get_imu_used order): the segment indices s_so3, s_r3, s_acc_bias, s_gyr_bias of its blocks
icc_status icco_get_imu_segments(const void* h, int32_t* seg4) {
  const Oracle& o = *O(h);
  for (const auto& b : o.blocks) {
    int32_t* r = seg4 + 4 * size_t(b.frame);
    if (b.type == BLK_ACCEL) {
      r[0] = int32_t((b.params[0].ptr - o.so3.data()) / 4); r[1] = int32_t((b.params[SPLINE_N].ptr - o.r3.data()) / 3);
      r[2] = int32_t((b.params[2 * SPLINE_N].ptr - o.ba.data()) / 3);
    } else if (b.type == BLK_GYRO) r[3] = int32_t((b.params[SPLINE_N].ptr - o.bg.data()) / 3);
  }
  return ICC_OK;
}

}  // extern "C"
