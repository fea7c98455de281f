// PINHOLE_RATIONAL (OpenCV's rational polynomial model, model id 9) in the oracle's templated form, test infrastructure only.
// oracle/oracle_math.hpp states the reference's camera models and stays as it is; this header states the extension from OpenCV's
// published projectPoints equations, scalar-templated so that the oracle's Jet type differentiates it.
//
// [f, ar, skew, cx, cy, k1, k2, k3, t1, t2, k4, k5, k6]: (xn, yn) = (x, y) / z, s = xn^2 + yn^2, R = N(s) / M(s),
// dx = xn R + 2 t1 xn yn + t2 (s + 2 xn^2), dy = yn R + t1 (s + 2 yn^2) + 2 t2 xn yn, u = f dx + skew dy + cx, v = f ar dy + cy.
// The domain (z > 0, s below the first fold or pole of r R(r^2)) is the product's and is not restated here.
#pragma once
#include "../../oracle/oracle_math.hpp"

namespace icco {

constexpr int PINHOLE_RATIONAL = 9;
constexpr int RATIONAL_N = 13;

template <class T> void rational_project(const T* k, const T* p, T* px) {
  const T xn = p[0] / p[2], yn = p[1] / p[2];
  const T s = xn * xn + yn * yn;
  const T N = 1.0 + s * (k[5] + s * (k[6] + s * k[7]));
  const T M = 1.0 + s * (k[10] + s * (k[11] + s * k[12]));
  const T R = N / M;
  const T dx = xn * R + 2.0 * k[8] * xn * yn + k[9] * (s + 2.0 * xn * xn);
  const T dy = yn * R + k[8] * (s + 2.0 * yn * yn) + 2.0 * k[9] * xn * yn;
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
}

}  // namespace icco

// ---- the CPU oracle's hook (rational_oracle.cpp) ----------------------------------------------------------------------------------------
// The oracle keeps ten intrinsics per camera.  PINHOLE_RATIONAL's first ten are its own ([f, ar, skew, cx, cy, k1, k2, k3, t1, t2]); the
// denominator k4, k5, k6 is held here, constant, set through rational_oracle_set_denominator.
namespace icco {
inline double g_rational_den[3] = {0.0, 0.0, 0.0};

// The domain, restated by sampling: z > 0 and, for every sigma in (0, s], M(sigma) > 0 and d(r R(r^2)) / dr > 0, i.e.
// h(sigma) = N M + 2 sigma (N' M - N M') > 0, checked in long double at 4096 points of (0, s] and at s itself.
inline bool rational_oracle_in_domain(const double* k, long double s) {
  const long double k1 = k[5], k2 = k[6], k3 = k[7], k4 = g_rational_den[0], k5 = g_rational_den[1], k6 = g_rational_den[2];
  for (int i = 1; i <= 4096; ++i) {
    const long double x = s * i / 4096;
    const long double N = 1 + x * (k1 + x * (k2 + x * k3)), M = 1 + x * (k4 + x * (k5 + x * k6));
    const long double dN = k1 + x * (2 * k2 + 3 * k3 * x), dM = k4 + x * (2 * k5 + 3 * k6 * x);
    if (!(M > 0) || !(N * M + 2 * x * (dN * M - N * dM) > 0)) return false;
  }
  return true;
}

template <class T> inline double scalar_part(const T& v) { return v.a; }
inline double scalar_part(double v) { return v; }

template <class T> inline bool rational_oracle_project(const T* k10, const T* p, T* px) {
  T k[RATIONAL_N];
  for (int i = 0; i < 10; ++i) k[i] = k10[i];
  for (int i = 0; i < 3; ++i) k[10 + i] = T(g_rational_den[i]);
  const double z = scalar_part(p[2]);
  if (!(z > 0.0)) { px[0] = T(0.0); px[1] = T(0.0); return false; }
  const double xn = scalar_part(p[0]) / z, yn = scalar_part(p[1]) / z;
  double kd[10];
  for (int i = 0; i < 10; ++i) kd[i] = scalar_part(k10[i]);
  if (!rational_oracle_in_domain(kd, (long double)xn * xn + (long double)yn * yn)) { px[0] = T(0.0); px[1] = T(0.0); return false; }
  rational_project<T>(k, p, px);
  return true;
}
}  // namespace icco
