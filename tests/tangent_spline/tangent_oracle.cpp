// Oracle of the spline solve's local tangent reprojection error (ICC_REPROJ_ERROR_TANGENT), for tests/test_tangent_spline.py.
//
// The CPU oracle (oracle/icc_oracle.cpp) is a fixed reference of the reference's pixel functor and stays as it is.  This file compiles
// it once more, unchanged, into a library of its own and swaps its vision functor for one that can also score corners against bearings:
//   * `rs_reprojection` (the oracle's RSReprojectionCostFunctorSplit) is renamed to `rs_reprojection_pixel` at its definition only: the
//     function-like macro matches `rs_reprojection(` but not the call `rs_reprojection<T>(`, which then resolves to the dispatcher below;
//   * the dispatcher runs the pixel functor, or the tangent one for an oracle that icco_set_tangent_bearings has given bearings;
//   * `icco_destroy` is wrapped the same way, so that a freed oracle's bearings never reach a later oracle at the same address.
// Everything else (problem assembly, autodiff Jacobians, local parameterisations, the LM driver) is the oracle's own code.  The tests
// supply the bearings from the NumPy camera models (wide_angle_support.oracle_bearings), never from the product.
#include <map>
#include <vector>

namespace {
struct Oracle;
struct Block;
template <class T> void rs_reprojection(const Oracle& o, const Block& b, const T* const* P, T* res);
}  // namespace

#define rs_reprojection(...) rs_reprojection_pixel(__VA_ARGS__)
#define icco_destroy(...) icco_destroy_pixel(__VA_ARGS__)
#include "../../oracle/icc_oracle.cpp"
#undef rs_reprojection
#undef icco_destroy

namespace {

// per oracle: unit bearing (3 per corner of icco_set_frames), whether it exists, pixels per tangent unit.  Written only between
// evaluations (from the caller's thread), read by the evaluation workers.
struct TangentMeas { std::vector<double> b; std::vector<int> ok; double s = 0.0; };
std::map<const Oracle*, TangentMeas> g_tangent;

// r = s (e1.p, e2.p) / (b.p) with the right-handed tangent basis of b (Duff et al., "Building an orthonormal basis, revisited", JCGT 2017);
// no bearing: 0; b.p <= 0: the failed-projection constant 1e10 of the pixel functor
template <class T>
void rs_tangent(const Oracle& o, const TangentMeas& M, const Block& blk, const T* const* P, T* res) {
  const int N2 = 2 * SPLINE_N;
  SE3T<T> T_i_c{{P[N2][0], P[N2][1], P[N2][2], P[N2][3]}, {P[N2][4], P[N2][5], P[N2][6]}};
  const T line_delay = P[N2 + 1][0];
  const Frame& f = o.frames[blk.frame];
  for (int c = f.c0; c < f.c1; ++c) {
    const int i = c - f.c0;
    const double oy = o.uv[2 * c + 1];
    const T y_coord = T(oy) * line_delay;
    Q4<T> R_w_i;
    evaluate_lie_so3<SPLINE_N, T>(P, T(blk.u_so3) + y_coord, T(o.inv_so3_dt), &R_w_i, nullptr);
    V3<T> t_w_i = evaluate_r3<SPLINE_N, 0, T>(P + SPLINE_N, T(blk.u_r3) + y_coord, T(o.inv_r3_dt));
    SE3T<T> T_c_w = se3_inv(se3_mul(SE3T<T>{R_w_i, t_w_i}, T_i_c));
    M3<T> R = so3_matrix(T_c_w.q);
    const T* X = P[N2 + 3 + i];
    T p[3];
    p[0] = (R.m[0][0] * X[0] + R.m[0][1] * X[1] + R.m[0][2] * X[2] + T_c_w.t.x * X[3]) / X[3];
    p[1] = (R.m[1][0] * X[0] + R.m[1][1] * X[1] + R.m[1][2] * X[2] + T_c_w.t.y * X[3]) / X[3];
    p[2] = (R.m[2][0] * X[0] + R.m[2][1] * X[1] + R.m[2][2] * X[2] + T_c_w.t.z * X[3]) / X[3];
    const double* b = &M.b[3 * size_t(c)];
    const double sg = b[2] < 0.0 ? -1.0 : 1.0, a = -1.0 / (sg + b[2]), bxy = b[0] * b[1] * a;
    const double e1[3] = {1.0 + sg * b[0] * b[0] * a, sg * bxy, -sg * b[0]}, e2[3] = {bxy, sg + b[1] * b[1] * a, -b[1]};
    const T bp = b[0] * p[0] + b[1] * p[1] + b[2] * p[2];
    if (!M.ok[c]) { res[2 * i] = T(0.0); res[2 * i + 1] = T(0.0); }
    else if (!(bp > 0.0)) { res[2 * i] = T(1e10); res[2 * i + 1] = T(1e10); }
    else {
      res[2 * i] = M.s * (e1[0] * p[0] + e1[1] * p[1] + e1[2] * p[2]) / bp;
      res[2 * i + 1] = M.s * (e2[0] * p[0] + e2[1] * p[1] + e2[2] * p[2]) / bp;
    }
  }
}

template <class T>
void rs_reprojection(const Oracle& o, const Block& b, const T* const* P, T* res) {
  const auto it = g_tangent.find(&o);
  if (it == g_tangent.end()) rs_reprojection_pixel<T>(o, b, P, res);
  else rs_tangent<T>(o, it->second, b, P, res);
}

}  // namespace

extern "C" {
// b[3n] / ok[n]: per corner of icco_set_frames its unit bearing and whether it exists; s: pixels per tangent unit.  b == NULL switches the
// oracle back to the pixel functor (e.g. for icco_get_mean_reprojection_error, which the product reports in pixels in either mode).
icc_status icco_set_tangent_bearings(void* h, int n, const double* b, const int32_t* ok, double s) {
  Oracle& o = *O(h);
  if (!b) { g_tangent.erase(&o); return ICC_OK; }
  if (!ok || n != int(o.point_ids.size())) { o.err = "one bearing per corner of set_frames"; return ICC_ERR_INVALID_ARGUMENT; }
  TangentMeas& M = g_tangent[&o];
  M.b.assign(b, b + 3 * size_t(n)); M.ok.assign(ok, ok + n); M.s = s;
  return ICC_OK;
}
void icco_destroy(void* h) { g_tangent.erase(O(h)); icco_destroy_pixel(h); }
}  // extern "C"
