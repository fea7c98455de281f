// The bearing math of the pose step's tangent residual (icc_bearing_math.cuh) compiled for the CPU, so that
// tests/test_wide_angle_poses.py can hold the product's un-projection and tangent error against the NumPy camera models.
#include "../../openimucameracalibrator_b200/csrc/icc_bearing_math.cuh"

using namespace icc;

extern "C" {
// unit bearings of n pixels: xyz[3n], ok[n]
void wa_unproject_bearings(int model, const double* k, int n, const double* uv, double* xyz, int* ok) {
  for (int i = 0; i < n; ++i) {
    V3 b;
    ok[i] = unproject_bearing(model, k, uv[2 * i], uv[2 * i + 1], b) ? 1 : 0;
    xyz[3 * i] = b.x; xyz[3 * i + 1] = b.y; xyz[3 * i + 2] = b.z;
  }
}
void wa_tangent_basis(const double* b, double* e1, double* e2) {
  V3 u, v; tangent_basis(v3(b[0], b[1], b[2]), u, v);
  e1[0] = u.x; e1[1] = u.y; e1[2] = u.z; e2[0] = v.x; e2[1] = v.y; e2[2] = v.z;
}
// tangent error of d = R(q) X + t against bearing b: r[2], front; J[12] = 2x6 pose Jacobian (right increment), P[6] = 2x3 board-point Jacobian
int wa_tangent_error(const double* b, const double* q_xyzw, const double* X, const double* t, double* r, double* J, double* P) {
  const Q4 q = q4(q_xyzw[0], q_xyzw[1], q_xyzw[2], q_xyzw[3]);
  const V3 Xv = v3(X[0], X[1], X[2]);
  const TangentErr E(qrot(q, Xv) + v3(t[0], t[1], t[2]), v3(b[0], b[1], b[2]));
  r[0] = E.r0; r[1] = E.r1;
  V3 P0, P1;
  tangent_jacobians(E, q, Xv, J, J + 6, P0, P1);
  P[0] = P0.x; P[1] = P0.y; P[2] = P0.z; P[3] = P1.x; P[4] = P1.y; P[5] = P1.z;
  return E.front() ? 1 : 0;
}
}
