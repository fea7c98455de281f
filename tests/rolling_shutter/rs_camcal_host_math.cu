// The rolling-shutter residual of the camera calibration (rs_camera_residual, icc_rolling_shutter_math.cuh) compiled for the CPU, so that
// tests/test_rolling_shutter_camera_calibration.py can hold its pose and intrinsic rows against central differences and against the
// global-shutter rows of camcal_accumulate_kernel, restated here from the same projection (project_with_k at R_cw (X - c)).
#include "../../openimucameracalibrator_b200/csrc/icc_rolling_shutter_math.cuh"

using namespace icc;

extern "C" {
// q = R_cw (x,y,z,w), c = camera centre, wu = (w, u), uv = the measured corner.  r[2], J[12] = 2x6 pose rows, Jk[20] = 2x10 intrinsic rows;
// returns the projection's ok flag.
int rs_camera_rows(int model, const double* k, const double* q_xyzw, const double* c, const double* X, const double* wu, double tau, const double* uv,
                   double* r, double* J, double* Jk) {
  RsMotion m; m.w = v3(wu[0], wu[1], wu[2]); m.u = v3(wu[3], wu[4], wu[5]);
  return rs_camera_residual(model, k, q4(q_xyzw[0], q_xyzw[1], q_xyzw[2], q_xyzw[3]), v3(c[0], c[1], c[2]), v3(X[0], X[1], X[2]), m, tau,
                            make_double2(uv[0], uv[1]), r[0], r[1], J, J + 6, Jk, Jk + 10) ? 1 : 0;
}
// the global-shutter rows of camcal_accumulate_kernel<JAC, false>
int gs_camera_rows(int model, const double* k, const double* q_xyzw, const double* c, const double* X, const double* uv, double* r, double* J, double* Jk) {
  const Q4 q = q4(q_xyzw[0], q_xyzw[1], q_xyzw[2], q_xyzw[3]);
  const V3 d = v3(X[0], X[1], X[2]) - v3(c[0], c[1], c[2]);
  ProjK pk;
  const Proj pr = project_with_k(model, k, qrot(q, d), true, &pk);
  r[0] = pr.u - uv[0]; r[1] = pr.v - uv[1];
  const V3 t0 = qrot_inv(q, v3(pr.J[0], pr.J[1], pr.J[2])), t1 = qrot_inv(q, v3(pr.J[3], pr.J[4], pr.J[5]));
  const V3 b0 = cross(d, t0), b1 = cross(d, t1);
  const double rows[12] = {b0.x, b0.y, b0.z, -t0.x, -t0.y, -t0.z, b1.x, b1.y, b1.z, -t1.x, -t1.y, -t1.z};
  for (int i = 0; i < 12; ++i) J[i] = rows[i];
  for (int i = 0; i < 20; ++i) Jk[i] = pk.Jk[i];
  return pr.ok ? 1 : 0;
}
}
