// Unit bearing vectors of pixels and the local tangent reprojection error of a predicted camera-frame point against a bearing:
// the measurement model of the pose step's opt-in wide-angle residual (ICC_POSE_ERROR_TANGENT, SURVEY.md §8(f) row f1).
//
// The default residual (the reference's BundleAdjustView) lives on the normalised plane z = 1, which cannot hold a ray 90 degrees or more
// off the optical axis, and a fixed pixel error there grows as ~1/cos^2(theta) towards the edge of a wide lens.  Here every corner is a
// unit ray b with an orthonormal tangent basis (e1, e2), and a predicted point d is scored by where it pierces the plane tangent to the
// unit sphere at b:  r = (e1.d, e2.d) / (b.d),  defined for b.d > 0.  With b = e_z, e1 = e_x, e2 = e_y this is exactly the normalised error
// of a corner at the principal point; |r| does not depend on the basis.
#pragma once
#include "icc_camera.cuh"

namespace icc {

// Orthonormal, right-handed (e1 x e2 = b) tangent basis of a unit vector, well conditioned for every b including -e_z
// (Duff et al., "Building an orthonormal basis, revisited", JCGT 2017).  b = e_z gives e1 = e_x, e2 = e_y exactly.
ICC_HD void tangent_basis(V3 b, V3& e1, V3& e2) {
  const double s = b.z < 0.0 ? -1.0 : 1.0, a = -1.0 / (s + b.z), c = b.x * b.y * a;
  e1 = v3(1.0 + s * b.x * b.x * a, s * c, -s * b.x);
  e2 = v3(c, s + b.y * b.y * a, -b.y);
}

// r = (e1.d, e2.d) / (b.d) and its rows a0 = d r0 / d d, a1 = d r1 / d d; front = (b.d > 0).  The pose Jacobian follows from d(d) =
// -R [X]x delta + dt (right increment), the board-point Jacobian from d(d) = R dX, exactly as for the normalised error in icc_pose.cu.
struct TangentErr {
  double r0, r1, is; V3 b;
  ICC_HD TangentErr(V3 d, V3 bb) : b(bb) {
    V3 e1, e2; tangent_basis(b, e1, e2);
    is = 1.0 / dot(b, d);
    r0 = dot(e1, d) * is; r1 = dot(e2, d) * is;
  }
  ICC_HD bool front() const { return is > 0.0; }
  ICC_HD void rows(V3& a0, V3& a1) const {
    V3 e1, e2; tangent_basis(b, e1, e2);
    a0 = is * (e1 - r0 * b); a1 = is * (e2 - r1 * b);
  }
};

// Jacobians of the tangent error of d = R X + t (R = R_cw, the quaternion q): J0 / J1 = rows of dr/d(delta, dt) for the right increment
// R exp(delta), t + dt, formed as pose_system forms them for the normalised error; P0 / P1 = rows of dr/dX for a board point X.
ICC_HD void tangent_jacobians(const TangentErr& E, Q4 q, V3 X, double J0[6], double J1[6], V3& P0, V3& P1) {
  V3 a0, a1; E.rows(a0, a1);
  P0 = qrot_inv(q, a0); P1 = qrot_inv(q, a1);
  const V3 b0 = cross(X, P0), b1 = cross(X, P1);
  J0[0] = b0.x; J0[1] = b0.y; J0[2] = b0.z; J0[3] = a0.x; J0[4] = a0.y; J0[5] = a0.z;
  J1[0] = b1.x; J1[1] = b1.y; J1[2] = b1.z; J1[3] = a1.x; J1[4] = a1.y; J1[5] = a1.z;
}

// The spline solve's local tangent reprojection error (ICC_REPROJ_ERROR_TANGENT) of a predicted camera-frame point pc against the corner's
// bearing, in the shape of a projection: (u, v) = s (e1.pc, e2.pc) / (b.pc) and J = s d(u, v)/d pc, so that every Jacobian column the
// evaluation kernels derive from the projection Jacobian stays as it is.  s = pixels per tangent unit at the image centre (tangent_scale);
// ok = the bearing could be formed (b_ok) and b.pc > 0.
ICC_HD Proj tangent_projection(double4 b4, bool b_ok, double s, V3 pc) {
  const TangentErr E(pc, v3(b4.x, b4.y, b4.z));
  V3 a0, a1; E.rows(a0, a1);
  Proj p;
  p.u = s * E.r0; p.v = s * E.r1;
  p.J[0] = s * a0.x; p.J[1] = s * a0.y; p.J[2] = s * a0.z; p.J[3] = s * a1.x; p.J[4] = s * a1.y; p.J[5] = s * a1.z;
  p.ok = b_ok && E.front();
  return p;
}

// sqrt(|det J0|), J0 = d(u, v)/d(x, y) of the model's projection at the principal ray (0, 0, 1): pixels per tangent unit at the image centre.
// It keeps the tangent residuals on the pixel scale that the IMU residuals' weights were tuned against (cov = I); 0 when the model
// cannot project the principal ray.
ICC_HD double tangent_scale(int model, const double* k, bool dispatch_fov) {
  const Proj p = project(model, k, v3(0.0, 0.0, 1.0), dispatch_fov);
  return p.ok ? sqrt(fabs(p.J[0] * p.J[4] - p.J[1] * p.J[3])) : 0.0;
}

// Unit ray b with project(b) within 1e-6 px of (px, py); false otherwise.  Pinhole, PinholeRadialTangential, FOV and DivisionUndistortion
// cannot see past 90 degrees: their ray is unproject_gn's normalised-plane point, normalised.  Fisheye, FisheyeRadtan, DoubleSphere,
// ExtendedUnified and OmniRadtan run
// damped Gauss-Newton on the sphere: the step lives in the tangent plane of the current b, its 2x2 Jacobian is the 2x3 projection Jacobian
// times (e1, e2), and the new ray is b + dx e1 + dy e2 renormalised.  Theia's Fisheye projects p and -p to the same pixel, so its ray is held
// in z > 0, and so is FisheyeRadtan's, whose domain is z > 0; the three unified models reach their whole forward domain, z <= 0 included (OmniRadtan: past 90 degrees for any xi > 0).
// Scaramuzza's model back-projects in closed form: the sensor point (u', v') = A^-1 (u - cx, v - cy) sees (u', v', F(rho)), for every
// rho = |(u', v')| below rho_max (beyond it the pixel is not the image of any point) and det A = c - d e != 0.
ICC_HD bool unproject_bearing(int model, const double* k, double px, double py, V3& b) {
  if (model == CAM_SCARAMUZZA) {
    const double det = k[1] - k[8] * k[2], du = px - k[3], dv = py - k[4];
    b = v3(0.0, 0.0, 1.0);
    if (!(det != 0.0) || !(k[0] > 0.0)) return false;
    const double up = (k[1] * du - k[2] * dv) / det, vp = (dv - k[8] * du) / det, rho = sqrt(up * up + vp * vp);
    if (!(rho < scaramuzza_rho_max(k))) return false;
    const V3 ray = v3(up, vp, scaramuzza_F(k, rho));
    b = (1.0 / sqrt(dot(ray, ray))) * ray;
    return true;
  }
  if (model != CAM_FISHEYE && model != CAM_FISHEYE_RADTAN && model != CAM_DOUBLE_SPHERE && model != CAM_EXTENDED_UNIFIED && model != CAM_OMNI_RADTAN) {
    double x = 0.0, y = 0.0;
    const bool good = unproject_gn(model, k, px, py, x, y);
    const double in = 1.0 / sqrt(x * x + y * y + 1.0);
    b = v3(x * in, y * in, in);
    return good;
  }
  // start: the linearised inverse at the principal ray gives a normalised-plane radius rho; read it as a stereographic one (theta = 2 atan(rho/2))
  const Proj p0 = project(model, k, v3(0.0, 0.0, 1.0), true);
  b = v3(0.0, 0.0, 1.0);
  if (!p0.ok) return false;
  {
    const double a = p0.J[0], bb = p0.J[1], c = p0.J[3], d = p0.J[4], det = a * d - bb * c;
    if (!(fabs(det) > 0.0)) return false;
    const double du = px - p0.u, dv = py - p0.v;
    const double x = (d * du - bb * dv) / det, y = (-c * du + a * dv) / det, rho = sqrt(x * x + y * y);
    if (rho > 0.0) {
      double th = 2.0 * atan(0.5 * rho);
      if (model == CAM_FISHEYE || model == CAM_FISHEYE_RADTAN) th = fmin(th, 1.5);
      const double s = sin(th) / rho;
      b = v3(x * s, y * s, cos(th));
    }
  }
  Proj p = project(model, k, b, true);
  for (int s = 0; s < 60 && !p.ok; ++s) { b = v3(0.5 * b.x, 0.5 * b.y, b.z + 0.5 * (1.0 - b.z)); b = (1.0 / sqrt(dot(b, b))) * b; p = project(model, k, b, true); }
  if (!p.ok) return false;
  double ru = p.u - px, rv = p.v - py, e = ru * ru + rv * rv;
  for (int it = 0; it < 60; ++it) {
    if (e < 1e-26) break;
    V3 e1, e2; tangent_basis(b, e1, e2);
    const double a = p.J[0] * e1.x + p.J[1] * e1.y + p.J[2] * e1.z, bb = p.J[0] * e2.x + p.J[1] * e2.y + p.J[2] * e2.z;
    const double c = p.J[3] * e1.x + p.J[4] * e1.y + p.J[5] * e1.z, d = p.J[3] * e2.x + p.J[4] * e2.y + p.J[5] * e2.z;
    const double det = a * d - bb * c;
    if (!(fabs(det) > 1e-300)) break;
    const double dx = -(d * ru - bb * rv) / det, dy = -(-c * ru + a * rv) / det;
    double t = 1.0; bool moved = false;
    for (int bt = 0; bt < 30; ++bt, t *= 0.5) {
      V3 bn = b + (t * dx) * e1 + (t * dy) * e2;
      bn = (1.0 / sqrt(dot(bn, bn))) * bn;
      if ((model == CAM_FISHEYE || model == CAM_FISHEYE_RADTAN) && !(bn.z > 0.0)) continue;
      const Proj pn = project(model, k, bn, true);
      if (!pn.ok) continue;
      const double r0 = pn.u - px, r1 = pn.v - py, en = r0 * r0 + r1 * r1;
      if (en < e) { b = bn; p = pn; ru = r0; rv = r1; e = en; moved = true; break; }
    }
    if (!moved) break;
  }
  return e < 1e-12;      // (1e-6 px)^2, the bar of unproject_gn
}

}  // namespace icc
