// Rolling-shutter model of the pose step (opt-in, icc_set_pose_rolling_shutter, SURVEY.md §8(f) row f1): every image row is exposed
// line_delay later than the one above it, so corner c of a view is seen tau_c = v_c * line_delay after the frame timestamp (v_c = its
// measured pixel row; the reference's RS functor uses the same rule, feature.y() * line_delay).  Over one readout the camera moves with
// constant camera-frame angular velocity w and linear velocity u, both at row 0, and a camera-frame point of the row-0 pose P0 = R X + t is
//   P(tau) = exp(-tau [w]x) (P0 - tau u).
// With w and u held fixed, dP/d(pose) = A(tau) dP0/d(pose), A = exp(-tau [w]x): the rows a0, a1 of either residual (normalised or tangent) become
// A^T a0, A^T a1 and the rest of the Jacobian is formed as before.  The velocities come from neighbouring views (rs_view_velocity).
#pragma once
#include "icc_bearing_math.cuh"

namespace icc {

struct RsMotion { V3 w, u; };   // camera-frame angular velocity (rad/s) and linear velocity (m/s) at row 0 of one view

ICC_HD Q4 rs_rotation(const RsMotion& m, double tau) { return so3_exp(-tau * m.w); }              // A(tau) = exp(-tau [w]x)
ICC_HD V3 rs_point(Q4 A, const RsMotion& m, double tau, V3 P0) { return qrot(A, P0 - tau * m.u); }  // P(tau)

// Residual of one corner against P(tau), P0 = R(q) X + t, and its 2x6 Jacobian rows for the right increment R exp(delta), t + dt (the
// parametrisation of pose_system).  xy: normalised point (front = P.z > 0); b: unit bearing with the tangent error (front = b.P > 0).
ICC_HD bool rs_pose_residual(double2 xy, Q4 q, V3 t, V3 X, const RsMotion& m, double tau, double& r0, double& r1, double J0[6], double J1[6]) {
  const Q4 A = rs_rotation(m, tau);
  const V3 P = rs_point(A, m, tau, qrot(q, X) + t);
  const double iz = 1.0 / P.z, u = P.x * iz, v = P.y * iz;
  r0 = u - xy.x; r1 = v - xy.y;
  const V3 a0 = qrot_inv(A, v3(iz, 0.0, -u * iz)), a1 = qrot_inv(A, v3(0.0, iz, -v * iz));
  const V3 b0 = cross(X, qrot_inv(q, a0)), b1 = cross(X, qrot_inv(q, a1));
  J0[0] = b0.x; J0[1] = b0.y; J0[2] = b0.z; J0[3] = a0.x; J0[4] = a0.y; J0[5] = a0.z;
  J1[0] = b1.x; J1[1] = b1.y; J1[2] = b1.z; J1[3] = a1.x; J1[4] = a1.y; J1[5] = a1.z;
  return P.z > 0.0;
}
ICC_HD bool rs_pose_residual(double4 b, Q4 q, V3 t, V3 X, const RsMotion& m, double tau, double& r0, double& r1, double J0[6], double J1[6]) {
  const Q4 A = rs_rotation(m, tau);
  const TangentErr E(rs_point(A, m, tau, qrot(q, X) + t), v3(b.x, b.y, b.z));
  r0 = E.r0; r1 = E.r1;
  V3 a0, a1; E.rows(a0, a1);
  a0 = qrot_inv(A, a0); a1 = qrot_inv(A, a1);
  const V3 b0 = cross(X, qrot_inv(q, a0)), b1 = cross(X, qrot_inv(q, a1));
  J0[0] = b0.x; J0[1] = b0.y; J0[2] = b0.z; J0[3] = a0.x; J0[4] = a0.y; J0[5] = a0.z;
  J1[0] = b1.x; J1[1] = b1.y; J1[2] = b1.z; J1[3] = a1.x; J1[4] = a1.y; J1[5] = a1.z;
  return E.front();
}

// Pixel residual of one corner of the camera calibration (icc_set_camcal_rolling_shutter) against P(tau), P0 = R_cw (X - c):
//   r = project(model, k, P(tau)) - uv.
// With J0 / J1 (nullable) the 2x6 rows for the right increment R_cw exp(delta) and the camera centre c, the columns of camcal_accumulate_kernel:
// (d x (R_cw^T A^T a), -(R_cw^T A^T a)), with a0, a1 the rows of the projection's 2x3 Jacobian at P(tau) and d = X - c.  With Jk0 / Jk1
// (nullable) the intrinsic rows d(u,v)/dk in Theia's order, max(10, camera_num_params(model)) entries each (zero beyond the model's
// parameters).  Returns the projection's ok flag.
ICC_HD bool rs_camera_residual(int model, const double* k, Q4 q, V3 c, V3 X, const RsMotion& m, double tau, double2 uv, double& r0, double& r1,
                               double J0[6], double J1[6], double* Jk0, double* Jk1) {
  const Q4 A = rs_rotation(m, tau);
  const V3 d = X - c;
  const V3 P = rs_point(A, m, tau, qrot(q, d));
  ProjK pk;
  const Proj pr = Jk0 ? project_with_k(model, k, P, true, &pk) : project(model, k, P, true);
  r0 = pr.u - uv.x; r1 = pr.v - uv.y;
  if (J0) {
    const V3 t0 = qrot_inv(q, qrot_inv(A, v3(pr.J[0], pr.J[1], pr.J[2]))), t1 = qrot_inv(q, qrot_inv(A, v3(pr.J[3], pr.J[4], pr.J[5])));
    const V3 b0 = cross(d, t0), b1 = cross(d, t1);
    J0[0] = b0.x; J0[1] = b0.y; J0[2] = b0.z; J0[3] = -t0.x; J0[4] = -t0.y; J0[5] = -t0.z;
    J1[0] = b1.x; J1[1] = b1.y; J1[2] = b1.z; J1[3] = -t1.x; J1[4] = -t1.y; J1[5] = -t1.z;
  }
  if (Jk0)
    for (int i = 0; i < 10 || i < camera_num_params(model); ++i) { Jk0[i] = pk.Jk[jk_at(0, i)]; Jk1[i] = pk.Jk[jk_at(1, i)]; }
  return pr.ok;
}

// Velocities of view f (pose R_f = R_wc(qf), camera centre pf) from two poses a (earlier, time ta) and b (later, tb) of the same camera:
//   w = R_f^T R_a Log(R_a^T R_b) / (tb - ta),   u = R_f^T (p_b - p_a) / (tb - ta).
// a and b are the previous and next neighbours (central difference), or one neighbour and f itself (one-sided).  Quaternions are q_wc.
ICC_HD RsMotion rs_view_velocity(Q4 qa, V3 pa, double ta, Q4 qb, V3 pb, double tb, Q4 qf) {
  const double idt = 1.0 / (tb - ta);
  RsMotion m;
  m.w = qrot_inv(qf, qrot(qa, idt * so3_log(qnormalized(qmul(qconj(qa), qb)))));
  m.u = qrot_inv(qf, idt * (pb - pa));
  return m;
}

}  // namespace icc
