// FISHEYE_RADIAL_TANGENTIAL (Kannala-Brandt with six radial and two tangential terms, model id 10) in the oracle's templated form, test
// infrastructure only.  oracle/oracle_math.hpp states the reference's camera models and stays as it is; this header states the extension
// from its published equations, scalar-templated so that the oracle's Jet type differentiates it.
//
// [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2]: r = |(x, y)|, theta = atan2(r, z),
// theta_d = theta (1 + k1 theta^2 + ... + k6 theta^12), (xr, yr) = (theta_d / r) (x, y) ((x, y) / z on the axis), s = xr^2 + yr^2,
// dx = xr + 2 t1 xr yr + t2 (s + 2 xr^2), dy = yr + t1 (s + 2 yr^2) + 2 t2 xr yr, u = f dx + skew dy + cx, v = f ar dy + cy.
// The domain (z > 0, d theta_d / d theta > 0 on (0, theta]) is restated by sampling in fisheye_radtan_oracle_in_domain.
#pragma once
#include "../../oracle/oracle_math.hpp"

namespace icco {

constexpr int FISHEYE_RADIAL_TANGENTIAL = 10;
constexpr int FISHEYE_RADTAN_N = 13;

template <class T> void fisheye_radtan_project(const T* k, const T* p, T* px) {
  const T r2 = p[0] * p[0] + p[1] * p[1];
  T xr, yr;
  if (!(r2 > 0.0)) {
    xr = p[0] / p[2]; yr = p[1] / p[2];
  } else {
    const T r = jsqrt(r2);
    const T th = jatan2(r, p[2]);
    const T t = th * th;
    const T thd = th * (1.0 + t * (k[5] + t * (k[6] + t * (k[7] + t * (k[8] + t * (k[9] + t * k[10]))))));
    xr = thd * p[0] / r; yr = thd * p[1] / r;
  }
  const T s = xr * xr + yr * yr;
  const T dx = xr + 2.0 * k[11] * xr * yr + k[12] * (s + 2.0 * xr * xr);
  const T dy = yr + k[11] * (s + 2.0 * yr * yr) + 2.0 * k[12] * xr * yr;
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
}

// The domain, restated by sampling: z > 0 and d theta_d / d theta = 1 + 3 k1 t + 5 k2 t^2 + ... + 13 k6 t^6 > 0 for every t in (0, theta^2],
// checked in long double at 4096 points of (0, theta^2] and at theta^2 itself.
inline bool fisheye_radtan_oracle_in_domain(const double* k, double x, double y, double z) {
  if (!(z > 0.0)) return false;
  const long double th = std::atan2(std::sqrt((long double)x * x + (long double)y * y), (long double)z), t2 = th * th;
  for (int i = 1; i <= 4096; ++i) {
    const long double t = t2 * i / 4096;
    const long double q = 1 + t * (3 * k[5] + t * (5 * k[6] + t * (7 * k[7] + t * (9 * k[8] + t * (11 * k[9] + t * 13 * k[10])))));
    if (!(q > 0)) return false;
  }
  return true;
}

}  // namespace icco
