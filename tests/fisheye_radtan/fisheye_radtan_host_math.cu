// The product's FISHEYE_RADIAL_TANGENTIAL camera math (icc_camera.cuh, icc_bearing_math.cuh, icc_rolling_shutter_math.cuh) compiled for
// the CPU, for tests/test_fisheye_radtan.py.  Intrinsic Jacobians come out as row-major 2 x ICC_MAX_INTRINSICS (Theia order).  Test
// infrastructure only.
#include "../../openimucameracalibrator_b200/csrc/icc_camera.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_bearing_math.cuh"
#include "../../openimucameracalibrator_b200/csrc/icc_rolling_shutter_math.cuh"

using namespace icc;

extern "C" {
int fhm_max_intrinsics() { return MAX_INTR; }
int fhm_num_params(int model) { return camera_num_params(model); }
int fhm_c_enum() { return ICC_CAM_FISHEYE_RADIAL_TANGENTIAL; }
int fhm_device_enum() { return CAM_FISHEYE_RADTAN; }
// out = [u, v, J (6), Jk (2 x MAX_INTR)]; returns ok | 2 when project() and project_with_k() agree bit for bit on value and point Jacobian
int fhm_project(int model, const double* k, const double* p, double* out) {
  ProjK pk;
  const Proj a = project_with_k(model, k, v3(p[0], p[1], p[2]), true, &pk);
  const Proj b = project(model, k, v3(p[0], p[1], p[2]), true);
  out[0] = a.u; out[1] = a.v;
  for (int i = 0; i < 6; ++i) out[2 + i] = a.J[i];
  for (int r = 0; r < 2; ++r) for (int c = 0; c < MAX_INTR; ++c) out[8 + MAX_INTR * r + c] = pk.Jk[jk_at(r, c)];
  int same = a.ok == b.ok && a.u == b.u && a.v == b.v;
  for (int i = 0; i < 6; ++i) same = same && a.J[i] == b.J[i];
  return (a.ok ? 1 : 0) | (same ? 2 : 0);
}
// the device's domain rule at theta^2 = t
int fhm_in_domain(const double* k, double t) { return fisheye_radtan_in_domain(k, t) ? 1 : 0; }
int fhm_unproject(int model, const double* k, double px, double py, double* xy) { double x = 0.0, y = 0.0; const bool ok = unproject_gn(model, k, px, py, x, y); xy[0] = x; xy[1] = y; return ok ? 1 : 0; }
int fhm_bearing(int model, const double* k, double px, double py, double* b3) { V3 b; const bool ok = unproject_bearing(model, k, px, py, b); b3[0] = b.x; b3[1] = b.y; b3[2] = b.z; return ok ? 1 : 0; }
// the camera calibration's rows at tau = 0 (a still camera): Jk0 / Jk1 with max(10, n_params) entries each
int fhm_camcal_rows(int model, const double* k, const double* q_xyzw, const double* c, const double* X, const double* uv, double* r, double* Jk0, double* Jk1) {
  RsMotion m; m.w = v3(0.0, 0.0, 0.0); m.u = v3(0.0, 0.0, 0.0);
  double J0[6], J1[6];
  return rs_camera_residual(model, k, q4(q_xyzw[0], q_xyzw[1], q_xyzw[2], q_xyzw[3]), v3(c[0], c[1], c[2]), v3(X[0], X[1], X[2]), m, 0.0, make_double2(uv[0], uv[1]),
                            r[0], r[1], J0, J1, Jk0, Jk1) ? 1 : 0;
}
}
