// Device camera-model "plugin surface": project a camera-frame point to pixels and return the analytic 2x3 Jacobian.
//
// Replaces theia::XCameraModel::CameraToPixelCoordinates<T>(intr, pt3, px) (pyTheiaSfM@69c3d37, external to
// the reference's repository) as dispatched at include/OpenCameraCalibrator/basalt_spline/ceres_calib_split_residuals.h:366-389,
// where the derivative came from Ceres Jets.  Intrinsic index order = Theia's InternalParametersIndex (see icc_b200.h).
// Return value = Theia's `bool` (false => the reference writes the constant 1e10 residual, quirk q12).
#pragma once
#include "icc_device_math.cuh"
#include "../../include/icc_b200.h"

namespace icc {

enum CameraModel { CAM_PINHOLE = 0, CAM_PINHOLE_RADTAN = 1, CAM_FISHEYE = 2, CAM_FOV = 3, CAM_DIVISION_UNDISTORTION = 4, CAM_DOUBLE_SPHERE = 5, CAM_EXTENDED_UNIFIED = 6,
                   CAM_OMNI_RADTAN = 7 /* extension: Kalibr's omni-radtan, no Theia counterpart */,
                   CAM_SCARAMUZZA = 8 /* extension: Scaramuzza's omnidirectional polynomial model (OCamCalib), no Theia counterpart */,
                   CAM_PINHOLE_RATIONAL = 9 /* extension: OpenCV's rational polynomial model (k1..k6, p1, p2), no Theia counterpart */,
                   CAM_FISHEYE_RADTAN = 10 /* extension: Kannala-Brandt with k1..k6 and tangential t1, t2 (Fisheye62), no Theia counterpart */ };

// Width of every intrinsic vector, buffer and Jacobian row in this library: the longest model's parameter count.
constexpr int MAX_INTR = ICC_MAX_INTRINSICS;

ICC_HD int camera_num_params(int model) {
  switch (model) { case CAM_PINHOLE: return 7; case CAM_PINHOLE_RADTAN: return 10; case CAM_FISHEYE: return 9; case CAM_FOV: return 5;
                   case CAM_DIVISION_UNDISTORTION: return 5; case CAM_DOUBLE_SPHERE: return 7; case CAM_EXTENDED_UNIFIED: return 7;
                   case CAM_OMNI_RADTAN: return 10; case CAM_SCARAMUZZA: return 9; case CAM_PINHOLE_RATIONAL: return 13;
                   case CAM_FISHEYE_RADTAN: return 13; default: return -1; }
}

// J is row-major 2x3: J[0..2] = d px / d(x,y,z), J[3..5] = d py / d(x,y,z).
// Jk (only filled when requested): d(u,v)/d intrinsics in Theia's parameter order, unused entries zero.  The first ten columns are
// row-major 2 x 10 in Jk[0..19]; the columns past ten (CAM_PINHOLE_RATIONAL's k4..k6, CAM_FISHEYE_RADTAN's k6, t1, t2) follow as row-major 2 x (MAX_INTR - 10): jk_at.
struct Proj { double u, v; double J[6]; bool ok; };
struct ProjK { double Jk[2 * MAX_INTR]; };
ICC_HD constexpr int jk_at(int row, int col) { return col < 10 ? 10 * row + col : 20 + (MAX_INTR - 10) * row + (col - 10); }

// final affine of the skewed models: u = f dx + s dy + cx, v = f ar dy + cy, given d(dx,dy)/dp
ICC_HD void affine_skew(const double* k, double dx, double dy, const double* Dd /*2x3*/, Proj& o) {
  const double f = k[0], fy = k[0] * k[1], s = k[2];
  o.u = f * dx + s * dy + k[3];
  o.v = fy * dy + k[4];
  for (int j = 0; j < 3; ++j) { o.J[j] = f * Dd[j] + s * Dd[3 + j]; o.J[3 + j] = fy * Dd[3 + j]; }
}
// intrinsic Jacobian of the skewed models: [f, ar, skew, cx, cy] columns + distortion columns idx[q] with d(dx,dy)/dk_q = (ddx[q], ddy[q])
ICC_HD void affine_skew_k(const double* k, double dx, double dy, int nd, const int* idx, const double* ddx, const double* ddy, ProjK& o) {
  for (int j = 0; j < 2 * MAX_INTR; ++j) o.Jk[j] = 0.0;
  o.Jk[0] = dx; o.Jk[10] = k[1] * dy;          // f
  o.Jk[11] = k[0] * dy;                        // aspect ratio
  o.Jk[2] = dy;                                // skew
  o.Jk[3] = 1.0; o.Jk[14] = 1.0;               // principal point
  for (int q = 0; q < nd; ++q) { o.Jk[jk_at(0, idx[q])] = k[0] * ddx[q] + k[2] * ddy[q]; o.Jk[jk_at(1, idx[q])] = k[0] * k[1] * ddy[q]; }
}

ICC_HD double unified_w(double alpha) { return alpha > 0.5 ? (1.0 - alpha) / alpha : alpha / (1.0 - alpha); }

// ---- Scaramuzza's omnidirectional polynomial model, [a0, c, e, cx, cy, a2, a3, a4, d] ------------------------------------------------
// A pixel's sensor point (u', v') = A^-1 (u - cx, v - cy), A = [[1, e], [d, c]], sees the ray (u', v', F(rho)), rho = |(u', v')|,
// F(rho) = a0 + a2 rho^2 + a3 rho^3 + a4 rho^4.  A point p = (x, y, z) at r = |(x, y)| projects to (u', v') = s (x, y), where s is the
// root of G(s) = F(r s) - z s on the branch where F(rho) / rho still falls: rho < rho_max, the first stationary point of F(rho) / rho.
ICC_HD double scaramuzza_F(const double* k, double rho) { return k[0] + rho * rho * (k[5] + rho * (k[6] + rho * k[7])); }

// Root of fn on [lo, hi], where fn(x, f, df) is increasing with f(lo) < 0 <= f(hi): Newton's method safeguarded by bisection, run until
// a step moves the iterate by at most an ulp or two.
template <class Fn> ICC_HD double bracketed_newton(const Fn& fn, double lo, double hi) {
  double x = 0.5 * (lo + hi);
  for (int it = 0; it < 100; ++it) {
    double f, df;
    fn(x, f, df);
    if (f < 0.0) lo = x; else if (f > 0.0) hi = x; else return x;
    double xn = x - f / df;
    if (!(xn > lo && xn < hi)) xn = 0.5 * (lo + hi);
    if (!(fabs(xn - x) > 2.5e-16 * fabs(xn))) return xn;
    x = xn;
  }
  return x;
}

// rho_max: the smallest positive root of q(rho) = rho F'(rho) - F(rho) = 3 a4 rho^4 + 2 a3 rho^3 + a2 rho^2 - a0 (q / rho^2 is the slope of
// F(rho) / rho), or +inf when q has none.  q(0) = -a0 < 0; q is monotone between its stationary points, the positive roots of
// q'(rho) / rho = 12 a4 rho^2 + 6 a3 rho + 2 a2, so the first piece on which q reaches 0 brackets the root.  A function of the intrinsics only.
ICC_HD double scaramuzza_rho_max(const double* k) {
  const double a0 = k[0], a2 = k[5], a3 = k[6], a4 = k[7];
  const auto fq = [&](double x, double& f, double& df) { f = x * x * (a2 + x * (2.0 * a3 + 3.0 * a4 * x)) - a0; df = x * (2.0 * a2 + x * (6.0 * a3 + 12.0 * a4 * x)); };
  double c0 = -1.0, c1 = -1.0;   // stationary points, ascending; <= 0 = none
  if (a4 != 0.0) {
    const double disc = 36.0 * a3 * a3 - 96.0 * a4 * a2;
    if (disc >= 0.0) {
      const double t = -0.5 * (6.0 * a3 + copysign(sqrt(disc), a3));
      if (t != 0.0) { const double x0 = t / (12.0 * a4), x1 = 2.0 * a2 / t; c0 = fmin(x0, x1); c1 = fmax(x0, x1); }
    }
  } else if (a3 != 0.0) {
    c1 = -a2 / (3.0 * a3);
  }
  double lo = 0.0, f, df;
  if (c0 > 0.0) { fq(c0, f, df); if (f >= 0.0) return bracketed_newton(fq, lo, c0); lo = c0; }
  if (c1 > 0.0) { fq(c1, f, df); if (f >= 0.0) return bracketed_newton(fq, lo, c1); lo = c1; }
  const double lead = a4 != 0.0 ? a4 : (a3 != 0.0 ? a3 : a2);   // q's leading coefficient has this sign
  if (!(lead > 0.0)) return INFINITY;
  double hi = fmax(2.0 * lo, 1.0);
  for (int i = 0; i < 2100; ++i) { fq(hi, f, df); if (f >= 0.0) break; lo = hi; hi *= 2.0; }
  return bracketed_newton(fq, lo, hi);
}

// The projection's scale s > 0 (G(s) = 0) of a point at distance r from the optical axis and depth z, and G_s = dG/ds < 0 there.
// The point is in the domain iff z / r > F(rho_max) / rho_max (z > 0 on the axis), the limit of F(rho) / rho standing in for rho_max = inf:
// 0 for a constant F, -inf otherwise.  There G falls through 0 exactly once on (0, rho_max / r): a bracket grown from a0 / |p| holds the root.
ICC_HD bool scaramuzza_scale(const double* k, double r, double z, double& s, double& gs) {
  const double a0 = k[0], a2 = k[5], a3 = k[6], a4 = k[7];
  const double rmax = scaramuzza_rho_max(k);
  const bool in = rmax < INFINITY ? z * rmax > r * scaramuzza_F(k, rmax) : (z > 0.0 || (r > 0.0 && !(a2 == 0.0 && a3 == 0.0 && a4 == 0.0)));
  const double pn = sqrt(r * r + z * z);
  if (!in || !(a0 > 0.0) || !(pn > 0.0)) return false;
  const auto fg = [&](double x, double& f, double& df) {   // -G and -G_s, increasing in s on the branch
    const double rho = r * x;
    f = z * x - (a0 + rho * rho * (a2 + rho * (a3 + rho * a4)));
    df = z - r * rho * (2.0 * a2 + rho * (3.0 * a3 + 4.0 * a4 * rho));
  };
  double lo = 0.0, hi = a0 / pn, f, df;
  bool bracketed = false;
  for (int i = 0; i < 128 && !bracketed; ++i) {
    if (r * hi >= rmax) { hi = rmax / r; bracketed = true; break; }
    fg(hi, f, df);
    if (f >= 0.0) bracketed = true; else { lo = hi; hi *= 4.0; }
  }
  if (!bracketed) return false;
  s = bracketed_newton(fg, lo, hi);
  fg(s, f, df);
  gs = -df;
  return true;
}

// ---- OpenCV's rational polynomial model, [f, ar, skew, cx, cy, k1, k2, k3, t1, t2, k4, k5, k6] -------------------------------------------
// R(s) = N(s) / M(s), N = 1 + k1 s + k2 s^2 + k3 s^3, M = 1 + k4 s + k5 s^2 + k6 s^3, s = xn^2 + yn^2.  A rational fit folds outside the
// field it was calibrated on, so the model is valid only for s < s_max: the first s > 0 at which the radial map r R(r^2) stops increasing,
// i.e. the first positive root of h = N M + 2 s (N' M - N M') (= M^2 d(r R) / dr) or of M (a pole); +inf when there is none.

// Whether the polynomial c[0] + c[1] x + ... + c[D] x^D (c[0] > 0) has no root in (0, s]: Descartes' rule of signs on the Moebius image
// q(y) = (1 + y)^D p((a + b y) / (1 + y)), whose positive roots are the roots of p in (a, b), bounds their number by the sign variations of
// q's coefficients, with equal parity.  0: (a, b) is clear; odd: a root; otherwise (a, b) is halved (Vincent's theorem: a small enough
// interval around simple roots counts exactly).  Left to right over (0, s]; a root cluster too tight to separate within the cap counts as a root.
template <int D> ICC_HD double poly_at(const double* c, double x) { double v = c[D]; for (int j = D - 1; j >= 0; --j) v = v * x + c[j]; return v; }
template <int D> ICC_HD int interval_sign_changes(const double* c, double a, double b) {
  double q[D + 1];
  for (int j = 0; j <= D; ++j) q[j] = c[j];
  for (int i = 0; i < D; ++i)                       // Taylor shift to a: q[j] = p^(j)(a) / j!
    for (int j = D - 1; j >= i; --j) q[j] += a * q[j + 1];
  double w = 1.0;
  for (int j = 1; j <= D; ++j) { w *= b - a; q[j] *= w; }   // p(a + (b - a) y)
  for (int j = 0; j < D / 2 + 1 && j < D - j; ++j) { const double t = q[j]; q[j] = q[D - j]; q[D - j] = t; }   // y^D p(1 / y)
  for (int i = 0; i < D; ++i)                       // Taylor shift by 1
    for (int j = D - 1; j >= i; --j) q[j] += q[j + 1];
  int v = 0; double prev = 0.0;
  for (int j = 0; j <= D; ++j) if (q[j] != 0.0) { if (prev != 0.0 && (q[j] > 0.0) != (prev > 0.0)) ++v; prev = q[j]; }
  return v;
}
template <int D> ICC_HD bool poly_root_free(const double* c, double s) {
  if (!(poly_at<D>(c, s) > 0.0)) return false;
  double a = 0.0, b = s;
  for (int it = 0; it < 200; ++it) {
    const int n = interval_sign_changes<D>(c, a, b);
    if (n == 0) {
      if (b >= s) return true;
      if (!(poly_at<D>(c, b) > 0.0)) return false;
      const double w = b - a;
      a = b; b = fmin(s, b + 2.0 * w);
      continue;
    }
    if (n & 1) return false;
    const double m = 0.5 * (a + b);
    if (!(m > a && m < b)) return false;
    b = m;
  }
  return false;
}
// The domain test at s >= 0: M(s) > 0 and s < s_max.
ICC_HD bool rational_in_domain(const double* k, double s) {
  const double k1 = k[5], k2 = k[6], k3 = k[7], k4 = k[10], k5 = k[11], k6 = k[12];
  if (!(1.0 + s * (k4 + s * (k5 + s * k6)) > 0.0)) return false;
  const double m[4] = {1.0, k4, k5, k6};
  // h = N M + 2 s (N' M - N M'): coefficient of s^j of N M is sum n_i m_(j-i), of s (N' M - N M') it is sum (i - (j - i)) n_i m_(j-i)
  const double n[4] = {1.0, k1, k2, k3};
  double h[7];
  for (int j = 0; j <= 6; ++j) {
    double acc = 0.0;
    for (int i = 0; i <= 3; ++i) if (j - i >= 0 && j - i <= 3) acc += (1.0 + 2.0 * (2 * i - j)) * n[i] * m[j - i];
    h[j] = acc;
  }
  return poly_root_free<3>(m, s) && poly_root_free<6>(h, s);
}

// ---- Kannala-Brandt with six radial and two tangential terms (Fisheye62), [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2] ---------
// theta = atan2(r, z), theta_d = theta P(theta^2), P(t) = 1 + k1 t + ... + k6 t^6, (xr, yr) = (theta_d / r) (x, y), then the tangential
// terms of PINHOLE_RADIAL_TANGENTIAL on (xr, yr) and the skewed affine.  Valid iff z > 0 and theta_d is still increasing on (0, theta]:
// d theta_d / d theta = Q(theta^2) = 1 + 3 k1 t + 5 k2 t^2 + ... + 13 k6 t^6 has no root in (0, theta^2] (t = theta^2 is the test's
// variable).  The tangential stage is not fold-checked, as for PINHOLE_RADIAL_TANGENTIAL.
__host__ __device__ inline __noinline__ bool fisheye_radtan_in_domain(const double* k, double t) {   // out of line: see project_fisheye_radtan
  const double q[7] = {1.0, 3.0 * k[5], 5.0 * k[6], 7.0 * k[7], 9.0 * k[8], 11.0 * k[9], 13.0 * k[10]};
  return poly_root_free<6>(q, t);
}

template <int MODEL, bool WITH_K = false>
ICC_HD Proj project_model(const double* k, V3 p, bool dispatch_fov, ProjK* pk = nullptr) {
  Proj o; o.ok = true;
  if (WITH_K) for (int j = 0; j < 2 * MAX_INTR; ++j) pk->Jk[j] = 0.0;
  if (MODEL == CAM_PINHOLE || MODEL == CAM_PINHOLE_RADTAN || MODEL == CAM_PINHOLE_RATIONAL) {
    if (MODEL == CAM_PINHOLE_RATIONAL && !(p.z > 0.0)) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double iz = 1.0 / p.z, xn = p.x * iz, yn = p.y * iz;
    const double r2 = xn * xn + yn * yn;
    double d, dd, dx, dy, a00, a01, a10, a11;   // a = d(dx,dy)/d(xn,yn)
    double iM = 1.0;                            // CAM_PINHOLE_RATIONAL: 1 / M
    if (MODEL == CAM_PINHOLE_RATIONAL && !rational_in_domain(k, r2)) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    if (MODEL == CAM_PINHOLE) {
      d = 1.0 + r2 * (k[5] + k[6] * r2); dd = k[5] + 2.0 * k[6] * r2;
      dx = xn * d; dy = yn * d;
      a00 = d + 2.0 * xn * xn * dd; a01 = 2.0 * xn * yn * dd; a10 = a01; a11 = d + 2.0 * yn * yn * dd;
    } else {
      const double k1 = k[5], k2 = k[6], k3 = k[7], t1 = k[8], t2 = k[9];
      d = 1.0 + r2 * (k1 + r2 * (k2 + r2 * k3)); dd = k1 + r2 * (2.0 * k2 + 3.0 * k3 * r2);
      if (MODEL == CAM_PINHOLE_RATIONAL) {        // d = N / M, dd = (N' - d M') / M
        const double k4 = k[10], k5 = k[11], k6 = k[12];
        iM = 1.0 / (1.0 + r2 * (k4 + r2 * (k5 + r2 * k6)));
        d *= iM; dd = (dd - d * (k4 + r2 * (2.0 * k5 + 3.0 * k6 * r2))) * iM;
      }
      dx = xn * d + 2.0 * t1 * xn * yn + t2 * (r2 + 2.0 * xn * xn);
      dy = yn * d + 2.0 * t2 * xn * yn + t1 * (r2 + 2.0 * yn * yn);
      a00 = d + 2.0 * xn * xn * dd + 2.0 * t1 * yn + 6.0 * t2 * xn;
      a01 = 2.0 * xn * yn * dd + 2.0 * t1 * xn + 2.0 * t2 * yn;
      a10 = 2.0 * xn * yn * dd + 2.0 * t2 * yn + 2.0 * t1 * xn;
      a11 = d + 2.0 * yn * yn * dd + 2.0 * t2 * xn + 6.0 * t1 * yn;
    }
    // d(xn,yn)/dp = [[iz,0,-xn iz],[0,iz,-yn iz]]
    double Dd[6] = {a00 * iz, a01 * iz, -(a00 * xn + a01 * yn) * iz, a10 * iz, a11 * iz, -(a10 * xn + a11 * yn) * iz};
    affine_skew(k, dx, dy, Dd, o);
    if (WITH_K) {
      if (MODEL == CAM_PINHOLE) { const int idx[2] = {5, 6}; const double ddx[2] = {xn * r2, xn * r2 * r2}, ddy[2] = {yn * r2, yn * r2 * r2}; affine_skew_k(k, dx, dy, 2, idx, ddx, ddy, *pk); }
      else if (MODEL == CAM_PINHOLE_RADTAN) { const int idx[5] = {5, 6, 7, 8, 9};
             const double ddx[5] = {xn * r2, xn * r2 * r2, xn * r2 * r2 * r2, 2.0 * xn * yn, r2 + 2.0 * xn * xn}, ddy[5] = {yn * r2, yn * r2 * r2, yn * r2 * r2 * r2, r2 + 2.0 * yn * yn, 2.0 * xn * yn};
             affine_skew_k(k, dx, dy, 5, idx, ddx, ddy, *pk); }
      else {   // dR/dk_i = s^i / M (k1..k3), -R s^i / M (k4..k6)
        const int idx[8] = {5, 6, 7, 8, 9, 10, 11, 12};
        const double ddx[8] = {xn * r2 * iM, xn * r2 * r2 * iM, xn * r2 * r2 * r2 * iM, 2.0 * xn * yn, r2 + 2.0 * xn * xn, -xn * d * r2 * iM, -xn * d * r2 * r2 * iM, -xn * d * r2 * r2 * r2 * iM};
        const double ddy[8] = {yn * r2 * iM, yn * r2 * r2 * iM, yn * r2 * r2 * r2 * iM, r2 + 2.0 * yn * yn, 2.0 * xn * yn, -yn * d * r2 * iM, -yn * d * r2 * r2 * iM, -yn * d * r2 * r2 * r2 * iM};
        affine_skew_k(k, dx, dy, 8, idx, ddx, ddy, *pk);
      }
    }
  } else if (MODEL == CAM_FISHEYE) {
    const double r2 = p.x * p.x + p.y * p.y;
    if (r2 < 1e-8) {
      double Dd[6] = {1, 0, 0, 0, 1, 0};
      affine_skew(k, p.x, p.y, Dd, o);
      if (WITH_K) affine_skew_k(k, p.x, p.y, 0, nullptr, nullptr, nullptr, *pk);
    } else {
      const double r = sqrt(r2), az = fabs(p.z), sg = p.z < 0.0 ? -1.0 : 1.0;
      const double th = atan2(r, az), th2 = th * th;
      const double thd = th * (1.0 + th2 * (k[5] + th2 * (k[6] + th2 * (k[7] + th2 * k[8]))));
      const double dthd = 1.0 + th2 * (3.0 * k[5] + th2 * (5.0 * k[6] + th2 * (7.0 * k[7] + th2 * 9.0 * k[8])));
      const double rho2 = r2 + p.z * p.z;
      const double g = thd / r;
      // dg/dx = (dthd * az/rho2 * x/r) / r - thd x / r^3 ; dg/dz = -dthd * sign(z) / rho2
      const double common = (dthd * az / rho2 - g) / r2;
      const double gx = common * p.x, gy = common * p.y, gz = -dthd * sg / rho2;
      double Dd[6] = {sg * (g + p.x * gx), sg * (p.x * gy), sg * (p.x * gz), sg * (p.y * gx), sg * (g + p.y * gy), sg * (p.y * gz)};
      affine_skew(k, sg * g * p.x, sg * g * p.y, Dd, o);
      if (WITH_K) { const int idx[4] = {5, 6, 7, 8}; const double t3 = th * th2, ex = sg * p.x / r, ey = sg * p.y / r;   // d theta_d / d k_i = theta^(2i+1)
                    const double ddx[4] = {t3 * ex, t3 * th2 * ex, t3 * th2 * th2 * ex, t3 * th2 * th2 * th2 * ex}, ddy[4] = {t3 * ey, t3 * th2 * ey, t3 * th2 * th2 * ey, t3 * th2 * th2 * th2 * ey};
                    affine_skew_k(k, sg * g * p.x, sg * g * p.y, 4, idx, ddx, ddy, *pk); }
    }
  } else if (MODEL == CAM_FOV) {
    if (!dispatch_fov) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double iz = 1.0 / p.z, xn = p.x * iz, yn = p.y * iz;
    const double r2 = xn * xn + yn * yn, om = k[4];
    double s, ds_r;  // s(r), (ds/dr)/r
    if (om * om < 1e-10) { s = 1.0; ds_r = 0.0; }
    else if (r2 < 1e-10) { s = 2.0 * tan(0.5 * om) / om; ds_r = 0.0; }
    else {
      const double r = sqrt(r2), T = tan(0.5 * om), at = atan(2.0 * r * T);
      s = at / (om * r);
      ds_r = ((2.0 * T / (1.0 + 4.0 * r2 * T * T)) * r - at) / (om * r2) / r;
    }
    const double a00 = s + xn * xn * ds_r, a01 = xn * yn * ds_r, a11 = s + yn * yn * ds_r;
    const double f = k[0], fy = k[0] * k[1];
    o.u = f * s * xn + k[2]; o.v = fy * s * yn + k[3];
    o.J[0] = f * a00 * iz; o.J[1] = f * a01 * iz; o.J[2] = -f * (a00 * xn + a01 * yn) * iz;
    o.J[3] = fy * a01 * iz; o.J[4] = fy * a11 * iz; o.J[5] = -fy * (a01 * xn + a11 * yn) * iz;
    if (WITH_K) {   // [f, ar, cx, cy, omega]
      double ds_om = 0.0;
      if (!(om * om < 1e-10)) {
        const double T = tan(0.5 * om), dT = 0.5 * (1.0 + T * T);
        if (r2 < 1e-10) ds_om = 2.0 * dT / om - 2.0 * T / (om * om);
        else { const double r = sqrt(r2), at = atan(2.0 * r * T); ds_om = (2.0 * r * dT / (1.0 + 4.0 * r2 * T * T)) / (om * r) - at / (om * om * r); }
      }
      pk->Jk[0] = s * xn; pk->Jk[10] = k[1] * s * yn; pk->Jk[11] = f * s * yn; pk->Jk[2] = 1.0; pk->Jk[13] = 1.0; pk->Jk[4] = f * ds_om * xn; pk->Jk[14] = fy * ds_om * yn;
    }
  } else if (MODEL == CAM_DIVISION_UNDISTORTION) {
    const double iz = 1.0 / p.z, f = k[0], fy = k[0] * k[1], kd = k[4];
    const double xu = f * p.x * iz, yu = fy * p.y * iz;
    const double r2 = xu * xu + yu * yu;
    const double den = 2.0 * kd * r2, inner = 1.0 - 4.0 * kd * r2;
    double s = 1.0, ds = 0.0;   // scale and d(scale)/d(r2)
    if (!(fabs(den) < 1e-15 || inner < 0.0)) {
      const double w = sqrt(inner);
      s = (1.0 - w) / den;
      ds = (den / w - (1.0 - w)) / (den * r2);
    }
    o.u = xu * s + k[2]; o.v = yu * s + k[3];
    const double a00 = s + 2.0 * xu * xu * ds, a01 = 2.0 * xu * yu * ds, a11 = s + 2.0 * yu * yu * ds;
    // d(xu)/dp = f [iz, 0, -x iz^2], d(yu)/dp = fy [0, iz, -y iz^2]
    const double xz = -xu * iz, yz = -yu * iz;
    o.J[0] = a00 * f * iz; o.J[1] = a01 * fy * iz; o.J[2] = a00 * xz + a01 * yz;
    o.J[3] = a01 * f * iz; o.J[4] = a11 * fy * iz; o.J[5] = a01 * xz + a11 * yz;
    if (WITH_K) {   // [f, ar, cx, cy, k]: xu, yu scale with f, yu with ar; d(scale)/dk = (den/w - (1-w)) / (k den)
      double dsk = 0.0;
      if (!(fabs(den) < 1e-15 || inner < 0.0)) { const double w = sqrt(inner); dsk = (den / w - (1.0 - w)) / (kd * den); }
      pk->Jk[0] = (a00 * xu + a01 * yu) / f; pk->Jk[10] = (a01 * xu + a11 * yu) / f;
      pk->Jk[1] = a01 * yu / k[1]; pk->Jk[11] = a11 * yu / k[1];
      pk->Jk[2] = 1.0; pk->Jk[13] = 1.0;
      pk->Jk[4] = xu * dsk; pk->Jk[14] = yu * dsk;
    }
  } else if (MODEL == CAM_DOUBLE_SPHERE) {
    const double xi = k[5], al = k[6];
    const double r2 = p.x * p.x + p.y * p.y;
    const double d1 = sqrt(r2 + p.z * p.z);
    const double w1 = unified_w(al), w2 = (w1 + xi) / sqrt(2.0 * w1 * xi + xi * xi + 1.0);
    if (p.z <= -w2 * d1) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double kk = xi * d1 + p.z;
    const double d2 = sqrt(r2 + kk * kk);
    const double nrm = al * d2 + (1.0 - al) * kk, in = 1.0 / nrm;
    // dk/dp = xi p/d1 + ez ; dd2/dp = (x, y, 0)/d2 + kk/d2 dk/dp ; dn = al dd2 + (1-al) dk
    const double kx = xi * p.x / d1, ky = xi * p.y / d1, kz = xi * p.z / d1 + 1.0;
    const double c = al * kk / d2 + (1.0 - al);
    const double nx = al * p.x / d2 + c * kx, ny = al * p.y / d2 + c * ky, nz = c * kz;
    const double dx = p.x * in, dy = p.y * in;
    double Dd[6] = {in - dx * nx * in, -dx * ny * in, -dx * nz * in, -dy * nx * in, in - dy * ny * in, -dy * nz * in};
    affine_skew(k, dx, dy, Dd, o);
    if (WITH_K) {   // d norm / d xi = d1 (al kk / d2 + 1 - al),  d norm / d alpha = d2 - kk ;  d(dx)/d. = -dx / norm * d norm
      const int idx[2] = {5, 6};
      const double dn[2] = {d1 * c, d2 - kk};
      const double ddx[2] = {-dx * in * dn[0], -dx * in * dn[1]}, ddy[2] = {-dy * in * dn[0], -dy * in * dn[1]};
      affine_skew_k(k, dx, dy, 2, idx, ddx, ddy, *pk);
    }
  } else if (MODEL == CAM_EXTENDED_UNIFIED) {
    const double al = k[5], be = k[6];
    const double r2 = p.x * p.x + p.y * p.y;
    const double rho = sqrt(be * r2 + p.z * p.z);
    const double nrm = al * rho + (1.0 - al) * p.z, in = 1.0 / nrm;
    if (p.z <= -unified_w(al) * rho) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double nx = al * be * p.x / rho, ny = al * be * p.y / rho, nz = al * p.z / rho + (1.0 - al);
    const double dx = p.x * in, dy = p.y * in;
    double Dd[6] = {in - dx * nx * in, -dx * ny * in, -dx * nz * in, -dy * nx * in, in - dy * ny * in, -dy * nz * in};
    affine_skew(k, dx, dy, Dd, o);
    if (WITH_K) {   // d norm / d alpha = rho - z,  d norm / d beta = alpha r2 / (2 rho)
      const int idx[2] = {5, 6};
      const double dn[2] = {rho - p.z, al * r2 / (2.0 * rho)};
      const double ddx[2] = {-dx * in * dn[0], -dx * in * dn[1]}, ddy[2] = {-dy * in * dn[0], -dy * in * dn[1]};
      affine_skew_k(k, dx, dy, 2, idx, ddx, ddy, *pk);
    }
  } else if (MODEL == CAM_OMNI_RADTAN) {   // [f, ar, skew, cx, cy, xi, k1, k2, t1, t2]: unit sphere, then the pinhole from -xi on the axis
    const double xi = k[5], k1 = k[6], k2 = k[7], t1 = k[8], t2 = k[9];
    const double d = sqrt(p.x * p.x + p.y * p.y + p.z * p.z);
    if (p.z <= -(xi <= 1.0 ? xi : 1.0 / xi) * d) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }   // EUCM's unified_w at alpha = xi / (1 + xi)
    const double in = 1.0 / (p.z + xi * d), mx = p.x * in, my = p.y * in;
    const double r2 = mx * mx + my * my;
    const double rad = 1.0 + r2 * (k1 + k2 * r2), drad = k1 + 2.0 * k2 * r2;
    const double dx = mx * rad + 2.0 * t1 * mx * my + t2 * (r2 + 2.0 * mx * mx);
    const double dy = my * rad + 2.0 * t2 * mx * my + t1 * (r2 + 2.0 * my * my);
    const double a00 = rad + 2.0 * mx * mx * drad + 2.0 * t1 * my + 6.0 * t2 * mx;   // a = d(dx,dy)/d(mx,my), symmetric
    const double a01 = 2.0 * mx * my * drad + 2.0 * t1 * mx + 2.0 * t2 * my;
    const double a11 = rad + 2.0 * my * my * drad + 2.0 * t2 * mx + 6.0 * t1 * my;
    // d(mx,my)/dp = in ([I2 | 0] - (mx, my)^T dn/dp), dn/dp = xi p / d + ez;  so d(dx,dy)/dp = in ([a | 0] - (a m) dn/dp^T)
    const double am0 = a00 * mx + a01 * my, am1 = a01 * mx + a11 * my;
    const double s = xi / d, nx = s * p.x, ny = s * p.y, nz = s * p.z + 1.0;
    double Dd[6] = {in * (a00 - am0 * nx), in * (a01 - am0 * ny), -in * am0 * nz, in * (a01 - am1 * nx), in * (a11 - am1 * ny), -in * am1 * nz};
    affine_skew(k, dx, dy, Dd, o);
    if (WITH_K) {   // d(mx,my)/d xi = -(mx,my) d / n
      const int idx[5] = {5, 6, 7, 8, 9};
      const double ddx[5] = {-am0 * d * in, mx * r2, mx * r2 * r2, 2.0 * mx * my, r2 + 2.0 * mx * mx};
      const double ddy[5] = {-am1 * d * in, my * r2, my * r2 * r2, r2 + 2.0 * my * my, 2.0 * mx * my};
      affine_skew_k(k, dx, dy, 5, idx, ddx, ddy, *pk);
    }
  } else if (MODEL == CAM_FISHEYE_RADTAN) {   // [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2]
    if (!(p.z > 0.0)) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double r2 = p.x * p.x + p.y * p.y, z2 = p.z * p.z, rho2 = r2 + z2, iz = 1.0 / p.z;
    // tr = theta / r and c = (Q z / rho^2 - g) / r^2 (g = theta_d / r: d g / d(x, y) = c (x, y)).  Near the axis (a^2 = r^2 / z^2 < 1e-8) both
    // from their series in a: theta / a = 1 - a^2 / 3 + a^4 / 5 (next term a^6 / 7 < 2e-25) and c = (2 k1 - 2 / 3) / z^3 (+ O(a^2), which
    // enters the Jacobian times x^2 <= r^2 only); exact on the axis itself.
    const bool axis = !(r2 > 1e-8 * z2);
    const double a2 = r2 * iz * iz;
    const double tr = axis ? (1.0 + a2 * (-1.0 / 3.0 + 0.2 * a2)) * iz : atan2(sqrt(r2), p.z) / sqrt(r2);
    const double t = tr * tr * r2;                                   // theta^2
    if (!fisheye_radtan_in_domain(k, t)) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double P = 1.0 + t * (k[5] + t * (k[6] + t * (k[7] + t * (k[8] + t * (k[9] + t * k[10])))));
    const double Q = 1.0 + t * (3.0 * k[5] + t * (5.0 * k[6] + t * (7.0 * k[7] + t * (9.0 * k[8] + t * (11.0 * k[9] + t * 13.0 * k[10])))));
    const double g = tr * P;
    const double c = axis ? (2.0 * k[5] - 2.0 / 3.0) * iz * iz * iz : (Q * p.z / rho2 - g) / r2;
    const double gz = -Q / rho2;
    const double xr = g * p.x, yr = g * p.y;
    const double M[6] = {g + p.x * p.x * c, p.x * p.y * c, p.x * gz, p.x * p.y * c, g + p.y * p.y * c, p.y * gz};   // d(xr, yr)/dp
    const double t1 = k[11], t2 = k[12], s = xr * xr + yr * yr;
    const double dx = xr + 2.0 * t1 * xr * yr + t2 * (s + 2.0 * xr * xr);
    const double dy = yr + t1 * (s + 2.0 * yr * yr) + 2.0 * t2 * xr * yr;
    const double a00 = 1.0 + 2.0 * t1 * yr + 6.0 * t2 * xr, a01 = 2.0 * t1 * xr + 2.0 * t2 * yr;   // a = d(dx, dy)/d(xr, yr), symmetric
    const double a11 = 1.0 + 2.0 * t2 * xr + 6.0 * t1 * yr;
    double Dd[6];
    for (int j = 0; j < 3; ++j) { Dd[j] = a00 * M[j] + a01 * M[3 + j]; Dd[3 + j] = a01 * M[j] + a11 * M[3 + j]; }
    affine_skew(k, dx, dy, Dd, o);
    if (WITH_K) {   // d(xr, yr)/dk_i = theta^(2i) (theta / r) (x, y) = t^i tr (x, y), through a; d(dx, dy)/dt1, dt2 directly
      const int idx[8] = {5, 6, 7, 8, 9, 10, 11, 12};
      double ddx[8], ddy[8], w = tr;
      for (int i = 0; i < 6; ++i) { w *= t; const double ex = w * p.x, ey = w * p.y; ddx[i] = a00 * ex + a01 * ey; ddy[i] = a01 * ex + a11 * ey; }
      ddx[6] = 2.0 * xr * yr; ddy[6] = s + 2.0 * yr * yr;
      ddx[7] = s + 2.0 * xr * xr; ddy[7] = 2.0 * xr * yr;
      affine_skew_k(k, dx, dy, 8, idx, ddx, ddy, *pk);
    }
  } else if (MODEL == CAM_SCARAMUZZA) {   // [a0, c, e, cx, cy, a2, a3, a4, d]: (u', v') = s (x, y), G(s) = 0; u = u' + e v' + cx, v = d u' + c v' + cy
    const double r = sqrt(p.x * p.x + p.y * p.y);
    double s, gs;
    if (!scaramuzza_scale(k, r, p.z, s, gs)) { o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
    const double c = k[1], e = k[2], d = k[8];
    const double up = s * p.x, vp = s * p.y;
    o.u = up + e * vp + k[3];
    o.v = d * up + c * vp + k[4];
    // implicit function theorem on G(s; p, k) = 0: ds = -dG / G_s, with dG/dx = x g, dG/dy = y g, dG/dz = -s, g = s^2 (2 a2 + 3 a3 rho + 4 a4 rho^2)
    const double rho = r * s, ig = -1.0 / gs;
    const double sg = s * s * (2.0 * k[5] + rho * (3.0 * k[6] + 4.0 * k[7] * rho)) * ig;
    const double sx = p.x * sg, sy = p.y * sg, sz = -s * ig;
    const double Du[3] = {s + p.x * sx, p.x * sy, p.x * sz}, Dv[3] = {p.y * sx, s + p.y * sy, p.y * sz};   // d(u', v')/dp
    for (int j = 0; j < 3; ++j) { o.J[j] = Du[j] + e * Dv[j]; o.J[3 + j] = d * Du[j] + c * Dv[j]; }
    if (WITH_K) {   // ds/da0 = -1 / G_s, ds/da_i = -rho^i / G_s
      const double wu = p.x + e * p.y, wv = d * p.x + c * p.y, rho2 = rho * rho;   // d(u, v)/ds
      pk->Jk[0] = wu * ig; pk->Jk[10] = wv * ig;
      pk->Jk[11] = vp;                        // c
      pk->Jk[2] = vp;                                   // e
      pk->Jk[3] = 1.0; pk->Jk[14] = 1.0;      // principal point
      pk->Jk[5] = wu * rho2 * ig; pk->Jk[15] = wv * rho2 * ig;
      pk->Jk[6] = wu * rho2 * rho * ig; pk->Jk[16] = wv * rho2 * rho * ig;
      pk->Jk[7] = wu * rho2 * rho2 * ig; pk->Jk[17] = wv * rho2 * rho2 * ig;
      pk->Jk[18] = up;                        // d
    }
  }
  return o;
}

// CAM_SCARAMUZZA and CAM_PINHOLE_RATIONAL out of line for the runtime dispatchers, behind one call: their root solves / root isolation
// stay out of the kernels that inline project() for every model
__host__ __device__ inline __noinline__ Proj project_out_of_line(int model, const double* k, V3 p) {
  return model == CAM_SCARAMUZZA ? project_model<CAM_SCARAMUZZA>(k, p, true) : project_model<CAM_PINHOLE_RATIONAL>(k, p, true);
}
__host__ __device__ inline __noinline__ Proj project_out_of_line_with_k(int model, const double* k, V3 p, ProjK* pk) {
  return model == CAM_SCARAMUZZA ? project_model<CAM_SCARAMUZZA, true>(k, p, true, pk) : project_model<CAM_PINHOLE_RATIONAL, true>(k, p, true, pk);
}
// CAM_FISHEYE_RADTAN out of line as well, on calls of its own from the dispatchers' default branch, with its domain test out of line in
// turn.  Of the arrangements tried, this is the one that leaves every kernel of the other models with no more registers or spills than
// before the model existed (-Xptxas -v); behind project_out_of_line it grew them.
__host__ __device__ inline __noinline__ Proj project_fisheye_radtan(const double* k, V3 p) { return project_model<CAM_FISHEYE_RADTAN>(k, p, true); }
__host__ __device__ inline __noinline__ Proj project_fisheye_radtan_with_k(const double* k, V3 p, ProjK* pk) { return project_model<CAM_FISHEYE_RADTAN, true>(k, p, true, pk); }

// Same dispatch, additionally returning d(u,v)/d(intrinsics) (CAM_INTRINSICS extension).
ICC_HD Proj project_with_k(int model, const double* k, V3 p, bool dispatch_fov, ProjK* pk) {
  switch (model) {
    case CAM_DIVISION_UNDISTORTION: return project_model<CAM_DIVISION_UNDISTORTION, true>(k, p, dispatch_fov, pk);
    case CAM_DOUBLE_SPHERE: return project_model<CAM_DOUBLE_SPHERE, true>(k, p, dispatch_fov, pk);
    case CAM_PINHOLE: return project_model<CAM_PINHOLE, true>(k, p, dispatch_fov, pk);
    case CAM_FISHEYE: return project_model<CAM_FISHEYE, true>(k, p, dispatch_fov, pk);
    case CAM_EXTENDED_UNIFIED: return project_model<CAM_EXTENDED_UNIFIED, true>(k, p, dispatch_fov, pk);
    case CAM_PINHOLE_RADTAN: return project_model<CAM_PINHOLE_RADTAN, true>(k, p, dispatch_fov, pk);
    case CAM_FOV: return project_model<CAM_FOV, true>(k, p, dispatch_fov, pk);
    case CAM_OMNI_RADTAN: return project_model<CAM_OMNI_RADTAN, true>(k, p, dispatch_fov, pk);
    case CAM_SCARAMUZZA: case CAM_PINHOLE_RATIONAL: return project_out_of_line_with_k(model, k, p, pk);
    default: {
      if (model == CAM_FISHEYE_RADTAN) return project_fisheye_radtan_with_k(k, p, pk);
      Proj o; o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; for (int j = 0; j < 2 * MAX_INTR; ++j) pk->Jk[j] = 0; return o; }
  }
}

// Runtime dispatch in the reference's order (residuals.h:366-389), then the extensions CAM_OMNI_RADTAN, CAM_SCARAMUZZA, CAM_PINHOLE_RATIONAL
// and CAM_FISHEYE_RADTAN.
ICC_HD Proj project(int model, const double* k, V3 p, bool dispatch_fov) {
  switch (model) {
    case CAM_DIVISION_UNDISTORTION: return project_model<CAM_DIVISION_UNDISTORTION>(k, p, dispatch_fov);
    case CAM_DOUBLE_SPHERE: return project_model<CAM_DOUBLE_SPHERE>(k, p, dispatch_fov);
    case CAM_PINHOLE: return project_model<CAM_PINHOLE>(k, p, dispatch_fov);
    case CAM_FISHEYE: return project_model<CAM_FISHEYE>(k, p, dispatch_fov);
    case CAM_EXTENDED_UNIFIED: return project_model<CAM_EXTENDED_UNIFIED>(k, p, dispatch_fov);
    case CAM_PINHOLE_RADTAN: return project_model<CAM_PINHOLE_RADTAN>(k, p, dispatch_fov);
    case CAM_FOV: return project_model<CAM_FOV>(k, p, dispatch_fov);
    case CAM_OMNI_RADTAN: return project_model<CAM_OMNI_RADTAN>(k, p, dispatch_fov);
    case CAM_SCARAMUZZA: case CAM_PINHOLE_RATIONAL: return project_out_of_line(model, k, p);
    default: {
      if (model == CAM_FISHEYE_RADTAN) return project_fisheye_radtan(k, p);
      Proj o; o.ok = false; o.u = o.v = 0; for (int j = 0; j < 6; ++j) o.J[j] = 0; return o; }
  }
}

// theia::Camera::PixelToNormalizedCoordinates(px) / z : solve project(x, y, 1) = px by damped Gauss-Newton
ICC_HD bool unproject_gn(int model, const double* k, double px, double py, double& xo, double& yo) {
  const Proj p0 = project(model, k, v3(0.0, 0.0, 1.0), true);
  if (!p0.ok) return false;
  double x, y;
  {
    const double a = p0.J[0], b = p0.J[1], c = p0.J[3], d = p0.J[4], det = a * d - b * c;
    if (!(fabs(det) > 0.0)) return false;
    const double du = px - p0.u, dv = py - p0.v;
    x = (d * du - b * dv) / det; y = (-c * du + a * dv) / det;
  }
  Proj p = project(model, k, v3(x, y, 1.0), true);
  for (int s = 0; s < 60 && !p.ok; ++s) { x *= 0.5; y *= 0.5; p = project(model, k, v3(x, y, 1.0), true); }   // outside the model's domain
  if (!p.ok) return false;
  double ru = p.u - px, rv = p.v - py, e = ru * ru + rv * rv;
  for (int it = 0; it < 50; ++it) {
    if (e < 1e-26) break;
    const double a = p.J[0], b = p.J[1], c = p.J[3], d = p.J[4], det = a * d - b * c;
    if (!(fabs(det) > 1e-300)) break;
    const double dx = -(d * ru - b * rv) / det, dy = -(-c * ru + a * rv) / det;
    double t = 1.0; bool moved = false;
    for (int bt = 0; bt < 30; ++bt, t *= 0.5) {
      const double xn = x + t * dx, yn = y + t * dy;
      const Proj pn = project(model, k, v3(xn, yn, 1.0), true);
      if (!pn.ok) continue;
      const double r0 = pn.u - px, r1 = pn.v - py, en = r0 * r0 + r1 * r1;
      if (en < e) { x = xn; y = yn; p = pn; ru = r0; rv = r1; e = en; moved = true; break; }
    }
    if (!moved) break;
  }
  xo = x; yo = y;
  return e < 1e-12;      // (1e-6 px)^2: anything worse did not converge
}

}  // namespace icc
