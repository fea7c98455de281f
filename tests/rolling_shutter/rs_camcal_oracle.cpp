// Oracle of the camera calibration with a rolling shutter (icc_set_camcal_rolling_shutter, fixed mode), for
// tests/test_rolling_shutter_camera_calibration.py.
//
// The CPU oracle (oracle/icc_oracle.cpp) stays as it is.  This file compiles it once more, unchanged, into a library of its own and swaps two of
// its functions for rolling-shutter versions, the way tests/tangent_spline/tangent_oracle.cpp swaps the spline solve's vision functor:
//   * `theia_reprojection_error` (the bundle adjustment's residual, autodiff over poses and intrinsics) and `point_residual` (the board-point
//     observation of BundleAdjustTracks) are renamed to *_gs at their definitions only: the function-like macros match `name(` but not the
//     calls `name<T>(`, which then resolve to the versions below;
//   * `icco_calibrate_camera` and `icco_destroy` are wrapped the same way.
// A corner is predicted from P(tau) = A (R_cw (X - c) - tau u), A = exp(-tau [w]x) a constant matrix (Rodrigues), tau = uv.y * line_delay,
// with (w, u) the fixed velocities of its view.  Everything else (problem assembly, Jet autodiff, the stages, the view filters, Ceres'
// trust-region loop, the point refinement) is the oracle's own code.
#include "../../oracle/oracle_math.hpp"

#include <algorithm>
#include <cmath>
#include <map>
#include <type_traits>
#include <vector>

namespace {
template <class T> bool theia_reprojection_error(int model, const T* ext, const T* intr, const double* X4, const double* feat, T* res);
template <class T> bool point_residual(bool normalized, int model, const double* intr, const icco::M3<double>& Rcw, const icco::V3<double>& cc, const T X[3],
                                       const double* meas, T r[2]);
}  // namespace

#define theia_reprojection_error(...) theia_reprojection_error_gs(__VA_ARGS__)
#define point_residual(...) point_residual_gs(__VA_ARGS__)
#define icco_calibrate_camera(...) icco_calibrate_camera_gs(__VA_ARGS__)
#define icco_destroy(...) icco_destroy_gs(__VA_ARGS__)
#include "../../oracle/icc_oracle.cpp"
#undef theia_reprojection_error
#undef point_residual
#undef icco_calibrate_camera
#undef icco_destroy

namespace {

struct RsShutter { double line_delay = 0.0; int nv = 0; std::vector<double> vel; };
std::map<const Oracle*, RsShutter> g_shutter;   // per oracle: icco_set_camcal_rolling_shutter

// The calibration in progress (the oracle's camera calibration is single-threaded).  The view of a corner comes from its position in the uv
// array; the camera centre of every view is recorded at each plain evaluation, so that a board-point observation (which carries the camera,
// not the view) finds its view: the last evaluation before BundleAdjustTracks is the final view filter's, at the poses it then holds fixed.
struct RsCall { const RsShutter* rs = nullptr; const double* uv = nullptr; const int32_t* off = nullptr; int nc = 0; std::vector<double> centre; };
RsCall g_call;

int view_of_corner(const double* feat) {
  const long c = (feat - g_call.uv) / 2;
  if (!g_call.rs || !g_call.uv || c < 0 || c >= g_call.nc) return -1;
  return int(std::upper_bound(g_call.off, g_call.off + g_call.rs->nv + 1, int32_t(c)) - g_call.off) - 1;
}
int view_of_centre(const Vd& cc) {
  for (int v = 0; v < g_call.rs->nv; ++v)
    if (g_call.centre[3 * v] == cc.x && g_call.centre[3 * v + 1] == cc.y && g_call.centre[3 * v + 2] == cc.z) return v;
  return -1;
}

// A = exp(-tau [w]x) as a row-major matrix (Rodrigues)
void rs_matrix(const double* w, double tau, double A[3][3]) {
  const double r[3] = {-tau * w[0], -tau * w[1], -tau * w[2]}, th = std::sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
  const double a = th > 1e-12 ? std::sin(th) / th : 1.0 - th * th / 6.0, b = th > 1e-12 ? (1.0 - std::cos(th)) / (th * th) : 0.5 - th * th / 24.0;
  const double K[3][3] = {{0.0, -r[2], r[1]}, {r[2], 0.0, -r[0]}, {-r[1], r[0], 0.0}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double kk = 0.0;
      for (int m = 0; m < 3; ++m) kk += K[i][m] * K[m][j];
      A[i][j] = (i == j ? 1.0 : 0.0) + a * K[i][j] + b * kk;
    }
}
template <class T> void rs_apply(const double* vel, double tau, const T P0[3], T P[3]) {
  double A[3][3];
  rs_matrix(vel, tau, A);
  const T d[3] = {P0[0] - tau * vel[3], P0[1] - tau * vel[4], P0[2] - tau * vel[5]};
  for (int i = 0; i < 3; ++i) P[i] = A[i][0] * d[0] + A[i][1] * d[1] + A[i][2] * d[2];
}

template <class T> bool theia_reprojection_error(int model, const T* ext, const T* intr, const double* X4, const double* feat, T* res) {
  const int v = view_of_corner(feat);
  if (v < 0) return theia_reprojection_error_gs<T>(model, ext, intr, X4, feat, res);
  if constexpr (std::is_same<T, double>::value) { for (int d = 0; d < 3; ++d) g_call.centre[3 * v + d] = ext[d]; }
  const T adj[3] = {T(X4[0]) - ext[0] * X4[3], T(X4[1]) - ext[1] * X4[3], T(X4[2]) - ext[2] * X4[3]};
  T rot[3], P[3], px[2];
  angle_axis_rotate(ext + 3, adj, rot);
  rs_apply<T>(&g_call.rs->vel[6 * (size_t)v], feat[1] * g_call.rs->line_delay, rot, P);
  const bool ok = project<T>(model, intr, P, px, true);
  res[0] = px[0] - feat[0]; res[1] = px[1] - feat[1];
  return ok;
}

template <class T> bool point_residual(bool normalized, int model, const double* intr, const M3<double>& Rcw, const Vd& cc, const T X[3], const double* meas, T r[2]) {
  const int v = (g_call.rs && !normalized) ? view_of_centre(cc) : -1;
  if (v < 0) return point_residual_gs<T>(normalized, model, intr, Rcw, cc, X, meas, r);
  const T d[3] = {X[0] - cc.x, X[1] - cc.y, X[2] - cc.z};
  T pc[3], P[3], k[10], px[2];
  for (int i = 0; i < 3; ++i) pc[i] = d[0] * Rcw.m[i][0] + d[1] * Rcw.m[i][1] + d[2] * Rcw.m[i][2];
  rs_apply<T>(&g_call.rs->vel[6 * (size_t)v], meas[1] * g_call.rs->line_delay, pc, P);
  for (int i = 0; i < 10; ++i) k[i] = T(intr[i]);
  if (!project<T>(model, k, P, px, true)) return false;
  r[0] = px[0] - meas[0]; r[1] = px[1] - meas[1];
  return true;
}

}  // namespace

extern "C" {
// line_delay_s = 0: the global shutter; > 0: w_u[6 n_views] = (w, u) per view, held fixed (the product's fixed mode).  frame_t_s is accepted
// for the product's signature and not read: the automatic mode is composed by the tests.
icc_status icco_set_camcal_rolling_shutter(void* h, double line_delay_s, int32_t n_views, const double* frame_t_s, const double* w_u) {
  Oracle& o = *O(h);
  if (!std::isfinite(line_delay_s) || line_delay_s < 0.0) { o.err = "line delay must be finite and >= 0"; return ICC_ERR_INVALID_ARGUMENT; }
  if (line_delay_s == 0.0) { g_shutter.erase(&o); return ICC_OK; }
  if (n_views <= 0 || !w_u) { o.err = "the oracle takes the view velocities (fixed mode)"; return ICC_ERR_INVALID_ARGUMENT; }
  RsShutter& S = g_shutter[&o];
  S.line_delay = line_delay_s; S.nv = n_views; S.vel.assign(w_u, w_u + 6 * (size_t)n_views);
  return ICC_OK;
}

icc_status icco_calibrate_camera(void* h, int model, int W, int Hh, int nv, const int32_t* off, const int32_t* ids, const double* uv,
                                 const double* q_init, const double* p_init, const int32_t* init_valid, double focal_init, double distortion_init,
                                 const icc_camcal_options* options, double* intr_out, double* q_out, double* p_out, double* err_out, int32_t* used_out,
                                 icc_camcal_summary* summary) {
  const auto it = g_shutter.find(O(h));
  if (it == g_shutter.end())
    return icco_calibrate_camera_gs(h, model, W, Hh, nv, off, ids, uv, q_init, p_init, init_valid, focal_init, distortion_init, options, intr_out, q_out, p_out, err_out, used_out, summary);
  if (nv != it->second.nv || !off) { O(h)->err = "n_views differs from that of set_camcal_rolling_shutter"; return ICC_ERR_INVALID_ARGUMENT; }
  g_call.rs = &it->second; g_call.uv = uv; g_call.off = off; g_call.nc = off[nv]; g_call.centre.assign(3 * (size_t)nv, std::nan(""));
  const icc_status rc = icco_calibrate_camera_gs(h, model, W, Hh, nv, off, ids, uv, q_init, p_init, init_valid, focal_init, distortion_init, options, intr_out, q_out, p_out, err_out,
                                                 used_out, summary);
  g_call = RsCall{};
  return rc;
}

void icco_destroy(void* h) { g_shutter.erase(O(h)); icco_destroy_gs(h); }
}  // extern "C"
