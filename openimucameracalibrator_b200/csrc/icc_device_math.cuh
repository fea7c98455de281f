// Device-side FP64 Lie / spline helpers for the calibration kernels.
//
// What these replace in the reference (each evaluated there through ceres::Jet autodiff on CPU threads):
//   SO3 exp/log/product      third_party/Sophus/sophus/so3.hpp:247-290,326-339,584-620  (same branches, eps = 1e-10)
//   cumulative SO(3) spline  include/OpenCameraCalibrator/basalt_spline/ceres_spline_helper.h:101-187
//   R^3 spline               include/OpenCameraCalibrator/basalt_spline/ceres_spline_helper.h:198-220
//   blending matrices        include/OpenCameraCalibrator/basalt_spline/spline_common.h:67-133
// New here: closed-form right Jacobians (Jr, Jr^-1) used for the ANALYTIC knot Jacobians (the reference has none on
// its live path; the recipe is Sommer et al. CVPR'20, cf. basalt_spline/so3_spline.h:202-256,350-421, re-derived for
// right-multiplicative knot increments R_i <- R_i exp(eps) so that it equals Ceres' autodiff x LieLocalParameterization).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace icc {

#define ICC_HD __host__ __device__ __forceinline__
#define ICC_D __device__ __forceinline__

constexpr double kEps = 1e-10;  // Sophus::Constants<double>::epsilon()  (sophus/common.hpp:94)

struct V3 { double x, y, z; };
struct Q4 { double x, y, z, w; };   // Sophus / Eigen coefficient order
struct M3 { double m[9]; };         // row-major

ICC_HD V3 v3(double x, double y, double z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
ICC_HD V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
ICC_HD V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
ICC_HD V3 operator*(double s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
ICC_HD V3 operator-(V3 a) { return v3(-a.x, -a.y, -a.z); }
ICC_HD double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
ICC_HD V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
ICC_HD V3 fma3(double s, V3 a, V3 b) { return v3(fma(s, a.x, b.x), fma(s, a.y, b.y), fma(s, a.z, b.z)); }

ICC_HD Q4 q4(double x, double y, double z, double w) { Q4 q; q.x = x; q.y = y; q.z = z; q.w = w; return q; }
ICC_HD Q4 qmul(Q4 a, Q4 b) {
  return q4(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
ICC_HD Q4 qconj(Q4 a) { return q4(-a.x, -a.y, -a.z, a.w); }
ICC_HD Q4 qnormalized(Q4 a) { const double n = 1.0 / sqrt(a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w); return q4(a.x * n, a.y * n, a.z * n, a.w * n); }
// p' = q p q*   (so3.hpp:359-370)
ICC_HD V3 qrot(Q4 q, V3 p) {
  V3 qv = v3(q.x, q.y, q.z);
  V3 uv = cross(qv, p);
  uv = uv + uv;
  return p + q.w * uv + cross(qv, uv);
}
ICC_HD V3 qrot_inv(Q4 q, V3 p) { return qrot(qconj(q), p); }
ICC_HD M3 qmat(Q4 q) {
  const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  M3 R;
  R.m[0] = 1.0 - (tyy + tzz); R.m[1] = txy - twz;         R.m[2] = txz + twy;
  R.m[3] = txy + twz;         R.m[4] = 1.0 - (txx + tzz); R.m[5] = tyz - twx;
  R.m[6] = txz - twy;         R.m[7] = tyz + twx;         R.m[8] = 1.0 - (txx + tyy);
  return R;
}
ICC_HD V3 mul(const M3& A, V3 b) { return v3(A.m[0] * b.x + A.m[1] * b.y + A.m[2] * b.z, A.m[3] * b.x + A.m[4] * b.y + A.m[5] * b.z, A.m[6] * b.x + A.m[7] * b.y + A.m[8] * b.z); }
ICC_HD V3 mulT(const M3& A, V3 b) { return v3(A.m[0] * b.x + A.m[3] * b.y + A.m[6] * b.z, A.m[1] * b.x + A.m[4] * b.y + A.m[7] * b.z, A.m[2] * b.x + A.m[5] * b.y + A.m[8] * b.z); }

// SO3::exp (so3.hpp:584-620).  Also returns the right-Jacobian coefficients of phi = omega:
//   Jr(phi) = I - a [phi]x + b [phi]x^2,  a = (1-cos t)/t^2,  b = (t - sin t)/t^3
struct ExpOut { Q4 q; double a, b; };
ICC_HD ExpOut so3_exp_jr(V3 om) {
  ExpOut o;
  const double th2 = dot(om, om);
  double imag, real;
  if (th2 < kEps * kEps) {
    const double th4 = th2 * th2;
    imag = 0.5 - (1.0 / 48.0) * th2 + (1.0 / 3840.0) * th4;
    real = 1.0 - (1.0 / 8.0) * th2 + (1.0 / 384.0) * th4;
    o.a = 0.5 - th2 * (1.0 / 24.0);
    o.b = (1.0 / 6.0) - th2 * (1.0 / 120.0);
  } else {
    const double th = sqrt(th2);
    double s, c;
    sincos(0.5 * th, &s, &c);
    imag = s / th;
    real = c;
    if (th2 < 1e-6) {   // series: closed forms cancel catastrophically for tiny angles
      o.a = 0.5 - th2 * (1.0 / 24.0) + th2 * th2 * (1.0 / 720.0);
      o.b = (1.0 / 6.0) - th2 * (1.0 / 120.0) + th2 * th2 * (1.0 / 5040.0);
    } else {
      o.a = 2.0 * s * s / th2;                 // (1 - cos t) = 2 sin^2(t/2)
      o.b = (th - 2.0 * s * c) / (th2 * th);   // sin t = 2 sin(t/2) cos(t/2)
    }
  }
  o.q = q4(imag * om.x, imag * om.y, imag * om.z, real);
  return o;
}
ICC_HD Q4 so3_exp(V3 om) { return so3_exp_jr(om).q; }

// SO3::log, atan based (so3.hpp:247-290)
ICC_HD V3 so3_log(Q4 q) {
  const double n2 = q.x * q.x + q.y * q.y + q.z * q.z;
  double f;
  if (n2 < kEps * kEps) {
    f = 2.0 / q.w - (2.0 / 3.0) * n2 / (q.w * q.w * q.w);
  } else {
    const double n = sqrt(n2);
    if (fabs(q.w) < kEps) f = (q.w > 0.0 ? M_PI : -M_PI) / n;
    else f = 2.0 * atan(n / q.w) / n;
  }
  return v3(f * q.x, f * q.y, f * q.z);
}

// Jr^-1(phi) = I + 1/2 [phi]x + c [phi]x^2, c = 1/t^2 - (1 + cos t)/(2 t sin t)
ICC_HD M3 so3_jr_inv(V3 p) {
  const double th2 = dot(p, p);
  double c;
  if (th2 < 1e-6) c = (1.0 / 12.0) + th2 * (1.0 / 720.0) + th2 * th2 * (1.0 / 30240.0);
  else { const double th = sqrt(th2); double s, co; sincos(th, &s, &co); c = 1.0 / th2 - (1.0 + co) / (2.0 * th * s); }
  M3 J;
  const double xx = p.x * p.x, yy = p.y * p.y, zz = p.z * p.z, xy = p.x * p.y, xz = p.x * p.z, yz = p.y * p.z;
  // [p]x^2 = p p^T - |p|^2 I
  J.m[0] = 1.0 - c * (yy + zz); J.m[1] = -0.5 * p.z + c * xy;  J.m[2] = 0.5 * p.y + c * xz;
  J.m[3] = 0.5 * p.z + c * xy;  J.m[4] = 1.0 - c * (xx + zz); J.m[5] = -0.5 * p.x + c * yz;
  J.m[6] = -0.5 * p.y + c * xz; J.m[7] = 0.5 * p.x + c * yz;  J.m[8] = 1.0 - c * (xx + yy);
  return J;
}

// row-vector times Jr(phi):  w Jr = w - a (w x phi) + b ((w x phi) x phi)
ICC_HD V3 row_times_jr(V3 w, V3 phi, double a, double b) {
  const V3 wp = cross(w, phi);
  return w - a * wp + b * cross(wp, phi);
}

// ---- blending (spline_common.h:67-133).  Known-answer tables x120 (N = 6) / x2 (N = 3): SURVEY.md §8(a2). ----------
// cumulative coefficients lambda_1..5 (lambda_0 == 1) and their u-derivatives
ICC_HD void cum_coeffs6(double u, double lam[5], double dlam[5]) {
  const double k = 1.0 / 120.0;
  const double u2 = u * u, u3 = u2 * u, u4 = u2 * u2, u5 = u4 * u;
  lam[0] = k * (119.0 + 5.0 * u - 10.0 * u2 + 10.0 * u3 - 5.0 * u4 + u5);
  lam[1] = k * (93.0 + 55.0 * u - 30.0 * u2 - 10.0 * u3 + 15.0 * u4 - 4.0 * u5);
  lam[2] = k * (27.0 + 55.0 * u + 30.0 * u2 - 10.0 * u3 - 15.0 * u4 + 6.0 * u5);
  lam[3] = k * (1.0 + 5.0 * u + 10.0 * u2 + 10.0 * u3 + 5.0 * u4 - 4.0 * u5);
  lam[4] = k * u5;
  dlam[0] = k * (5.0 - 20.0 * u + 30.0 * u2 - 20.0 * u3 + 5.0 * u4);
  dlam[1] = k * (55.0 - 60.0 * u - 30.0 * u2 + 60.0 * u3 - 20.0 * u4);
  dlam[2] = k * (55.0 + 60.0 * u - 30.0 * u2 - 60.0 * u3 + 30.0 * u4);
  dlam[3] = k * (5.0 + 20.0 * u + 30.0 * u2 + 20.0 * u3 - 20.0 * u4);
  dlam[4] = k * (5.0 * u4);
}
// non-cumulative coefficients c_0..5 and u-derivatives of order 1 and 2
ICC_HD void coeffs6(double u, double c[6], double dc[6], double ddc[6]) {
  const double k = 1.0 / 120.0;
  const double u2 = u * u, u3 = u2 * u, u4 = u2 * u2, u5 = u4 * u;
  c[0] = k * (1.0 - 5.0 * u + 10.0 * u2 - 10.0 * u3 + 5.0 * u4 - u5);
  c[1] = k * (26.0 - 50.0 * u + 20.0 * u2 + 20.0 * u3 - 20.0 * u4 + 5.0 * u5);
  c[2] = k * (66.0 - 60.0 * u2 + 30.0 * u4 - 10.0 * u5);
  c[3] = k * (26.0 + 50.0 * u + 20.0 * u2 - 20.0 * u3 - 20.0 * u4 + 10.0 * u5);
  c[4] = k * (1.0 + 5.0 * u + 10.0 * u2 + 10.0 * u3 + 5.0 * u4 - 5.0 * u5);
  c[5] = k * u5;
  if (dc) {
    dc[0] = k * (-5.0 + 20.0 * u - 30.0 * u2 + 20.0 * u3 - 5.0 * u4);
    dc[1] = k * (-50.0 + 40.0 * u + 60.0 * u2 - 80.0 * u3 + 25.0 * u4);
    dc[2] = k * (-120.0 * u + 120.0 * u3 - 50.0 * u4);
    dc[3] = k * (50.0 + 40.0 * u - 60.0 * u2 - 80.0 * u3 + 50.0 * u4);
    dc[4] = k * (5.0 + 20.0 * u + 30.0 * u2 + 20.0 * u3 - 25.0 * u4);
    dc[5] = k * (5.0 * u4);
  }
  if (ddc) {
    ddc[0] = k * (20.0 - 60.0 * u + 60.0 * u2 - 20.0 * u3);
    ddc[1] = k * (40.0 + 120.0 * u - 240.0 * u2 + 100.0 * u3);
    ddc[2] = k * (-120.0 + 360.0 * u2 - 200.0 * u3);
    ddc[3] = k * (40.0 - 120.0 * u - 240.0 * u2 + 200.0 * u3);
    ddc[4] = k * (20.0 + 60.0 * u + 60.0 * u2 - 100.0 * u3);
    ddc[5] = k * (20.0 * u3);
  }
}
// second u-derivative of the cumulative coefficients and third of the non-cumulative ones (time-offset extension:
// angular acceleration and jerk of the spline)
ICC_HD void cum_coeffs6_dd(double u, double ddlam[5]) {
  const double k = 1.0 / 120.0, u2 = u * u, u3 = u2 * u;
  ddlam[0] = k * (-20.0 + 60.0 * u - 60.0 * u2 + 20.0 * u3);
  ddlam[1] = k * (-60.0 - 60.0 * u + 180.0 * u2 - 80.0 * u3);
  ddlam[2] = k * (60.0 - 60.0 * u - 180.0 * u2 + 120.0 * u3);
  ddlam[3] = k * (20.0 + 60.0 * u + 60.0 * u2 - 80.0 * u3);
  ddlam[4] = k * (20.0 * u3);
}
ICC_HD void coeffs6_ddd(double u, double dddc[6]) {
  const double k = 1.0 / 120.0, u2 = u * u;
  dddc[0] = k * (-60.0 + 120.0 * u - 60.0 * u2);
  dddc[1] = k * (120.0 - 480.0 * u + 300.0 * u2);
  dddc[2] = k * (720.0 * u - 600.0 * u2);
  dddc[3] = k * (-120.0 - 480.0 * u + 600.0 * u2);
  dddc[4] = k * (60.0 + 120.0 * u - 300.0 * u2);
  dddc[5] = k * (60.0 * u2);
}
ICC_HD void coeffs3_d(double u, double dc[3]) { dc[0] = u - 1.0; dc[1] = 1.0 - 2.0 * u; dc[2] = u; }
// bias spline, N = 3, non-cumulative:  rows x2 = [1 -2 1; 1 2 -2; 0 0 1]
ICC_HD void coeffs3(double u, double c[3]) {
  const double u2 = u * u;
  c[0] = 0.5 * (1.0 - 2.0 * u + u2);
  c[1] = 0.5 * (1.0 + 2.0 * u - 2.0 * u2);
  c[2] = 0.5 * u2;
}

}  // namespace icc
