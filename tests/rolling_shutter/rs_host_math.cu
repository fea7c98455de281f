// The rolling-shutter math of the pose step (icc_rolling_shutter_math.cuh) compiled for the CPU, so that
// tests/test_rolling_shutter_poses.py can hold the product's transform, residual rows and neighbour velocities against central differences.
#include "../../openimucameracalibrator_b200/csrc/icc_rolling_shutter_math.cuh"

using namespace icc;

extern "C" {
// residual of one corner seen at row time tau: meas = (x, y) normalised (tangent = 0) or a unit bearing (tangent = 1); q = R_cw (x,y,z,w),
// wu = (w, u).  r[2], J[12] = 2x6 pose Jacobian for the right increment; returns front.
int rs_residual(int tangent, const double* meas, const double* q_xyzw, const double* X, const double* t, const double* wu, double tau, double* r, double* J) {
  const Q4 q = q4(q_xyzw[0], q_xyzw[1], q_xyzw[2], q_xyzw[3]);
  RsMotion m; m.w = v3(wu[0], wu[1], wu[2]); m.u = v3(wu[3], wu[4], wu[5]);
  const V3 Xv = v3(X[0], X[1], X[2]), tv = v3(t[0], t[1], t[2]);
  const bool front = tangent ? rs_pose_residual(make_double4(meas[0], meas[1], meas[2], 0.0), q, tv, Xv, m, tau, r[0], r[1], J, J + 6)
                             : rs_pose_residual(make_double2(meas[0], meas[1]), q, tv, Xv, m, tau, r[0], r[1], J, J + 6);
  return front ? 1 : 0;
}
// P(tau) of a camera-frame point P0
void rs_transform(const double* P0, const double* wu, double tau, double* P) {
  RsMotion m; m.w = v3(wu[0], wu[1], wu[2]); m.u = v3(wu[3], wu[4], wu[5]);
  const V3 r = rs_point(rs_rotation(m, tau), m, tau, v3(P0[0], P0[1], P0[2]));
  P[0] = r.x; P[1] = r.y; P[2] = r.z;
}
// velocities of view f from poses a (ta) and b (tb): quaternions q_wc (x,y,z,w), positions p_wc; wu[6] = (w, u)
void rs_velocity(const double* qa, const double* pa, double ta, const double* qb, const double* pb, double tb, const double* qf, double* wu) {
  const RsMotion m = rs_view_velocity(q4(qa[0], qa[1], qa[2], qa[3]), v3(pa[0], pa[1], pa[2]), ta, q4(qb[0], qb[1], qb[2], qb[3]), v3(pb[0], pb[1], pb[2]), tb,
                                      q4(qf[0], qf[1], qf[2], qf[3]));
  wu[0] = m.w.x; wu[1] = m.w.y; wu[2] = m.w.z; wu[3] = m.u.x; wu[4] = m.u.y; wu[5] = m.u.z;
}
}
