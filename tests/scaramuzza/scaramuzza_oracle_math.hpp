// SCARAMUZZA (Scaramuzza's omnidirectional polynomial model as OCamCalib calibrates it, model id 8) for the CPU oracle, test infrastructure
// only.  oracle/oracle_math.hpp states the reference's camera models and stays as it is; this header states the extension model from its
// published equations in the same templated form, and dispatches to the oracle's own `project` for every other model.
//
// [a0, c, e, cx, cy, a2, a3, a4, d]: a point p at r = |(x, y)| projects to the sensor point s (x, y), s the root of
// G(s) = a0 - z s + a2 (r s)^2 + a3 (r s)^3 + a4 (r s)^4 below rho_max / r, then u = u' + e v' + cx, v = d u' + c v' + cy.  The root is
// found on the scalar parts alone (bisection in long double); one Newton step s - G(s) / G_s(s) taken in the Jet type then carries the
// exact first derivatives (the implicit function theorem), so the oracle's autodiff differentiates the model.
#pragma once
#include "../../oracle/oracle_math.hpp"

namespace icco {

constexpr int SCARAMUZZA = 8;

struct ScaraPoly { long double a0, a2, a3, a4; };
inline long double scara_F(const ScaraPoly& a, long double rho) { return a.a0 + a.a2 * rho * rho + a.a3 * rho * rho * rho + a.a4 * rho * rho * rho * rho; }
// q(rho) = rho F'(rho) - F(rho): the sign of the slope of F(rho) / rho
inline long double scara_q(const ScaraPoly& a, long double rho) { return 3 * a.a4 * rho * rho * rho * rho + 2 * a.a3 * rho * rho * rho + a.a2 * rho * rho - a.a0; }

// the root of q on [lo, hi] (q(lo) < 0 <= q(hi)) by bisection to the end of long double
inline long double scara_bisect_q(const ScaraPoly& a, long double lo, long double hi) {
  for (int i = 0; i < 400; ++i) { const long double m = 0.5L * (lo + hi); if (m <= lo || m >= hi) break; (scara_q(a, m) < 0 ? lo : hi) = m; }
  return 0.5L * (lo + hi);
}

// rho_max = the first positive root of q (inf when there is none): q is monotone between its stationary points, the positive roots of
// 12 a4 rho^2 + 6 a3 rho + 2 a2
inline long double scara_rho_max(const ScaraPoly& a) {
  long double st[2]; int n = 0;
  if (a.a4 != 0) {
    const long double disc = 36 * a.a3 * a.a3 - 96 * a.a4 * a.a2;
    if (disc >= 0) { const long double sq = std::sqrt(disc); st[n++] = (-6 * a.a3 - sq) / (24 * a.a4); st[n++] = (-6 * a.a3 + sq) / (24 * a.a4); }
  } else if (a.a3 != 0) {
    st[n++] = -a.a2 / (3 * a.a3);
  }
  if (n == 2 && st[0] > st[1]) std::swap(st[0], st[1]);
  long double lo = 0;
  for (int i = 0; i < n; ++i) {
    if (!(st[i] > lo)) continue;
    if (scara_q(a, st[i]) >= 0) return scara_bisect_q(a, lo, st[i]);
    lo = st[i];
  }
  const long double lead = a.a4 != 0 ? a.a4 : (a.a3 != 0 ? a.a3 : a.a2);
  if (!(lead > 0)) return HUGE_VALL;
  long double hi = lo > 0 ? 2 * lo : 1;
  while (scara_q(a, hi) < 0) { lo = hi; hi *= 2; }
  return scara_bisect_q(a, lo, hi);
}

// s with G(s) = 0 on the branch, false outside the domain z / r > F(rho_max) / rho_max (z > 0 on the axis; the limit of F(rho) / rho
// when rho_max = inf: 0 for a constant F, -inf otherwise)
inline bool scara_scale(const ScaraPoly& a, long double r, long double z, long double& s) {
  const long double rmax = scara_rho_max(a);
  const bool flat = a.a2 == 0 && a.a3 == 0 && a.a4 == 0;
  const bool in = std::isinf(rmax) ? (z > 0 || (r > 0 && !flat)) : z * rmax > r * scara_F(a, rmax);
  if (!in || !(a.a0 > 0)) return false;
  auto negG = [&](long double x) { return z * x - scara_F(a, r * x); };   // increasing on the branch
  const long double cap = r > 0 ? rmax / r : HUGE_VALL;
  long double lo = 0, hi = a.a0 / std::sqrt(r * r + z * z);
  for (int i = 0; i < 4000 && negG(hi) < 0; ++i) {
    if (hi >= cap) break;
    lo = hi; hi = std::min(2 * hi, cap);
  }
  if (!(negG(hi) >= 0) && !(hi >= cap)) return false;
  for (int i = 0; i < 400; ++i) { const long double m = 0.5L * (lo + hi); if (m <= lo || m >= hi) break; (negG(m) < 0 ? lo : hi) = m; }
  s = 0.5L * (lo + hi);
  return true;
}

template <class T> inline bool project_scaramuzza(const T* k, const T* p, T* px) {
  const ScaraPoly a{jval(k[0]), jval(k[5]), jval(k[6]), jval(k[7])};
  const double x = jval(p[0]), y = jval(p[1]), z = jval(p[2]);
  const double rv = std::sqrt(x * x + y * y);
  long double sl;
  if (!scara_scale(a, rv, z, sl)) return false;
  const double s = (double)sl, rho = rv * s;
  const double gs = -z + rv * rho * (2.0 * (double)a.a2 + 3.0 * (double)a.a3 * rho + 4.0 * (double)a.a4 * rho * rho);   // G_s < 0
  const T r2 = p[0] * p[0] + p[1] * p[1];
  const T r = r2 > 0.0 ? jsqrt(r2) : T(0.0);   // d(r^3)/dp = 3 r (x, y, 0) vanishes on the axis
  const T S(s);
  const T G = k[0] - p[2] * S + k[5] * r2 * S * S + k[6] * r2 * r * S * S * S + k[7] * r2 * r2 * S * S * S * S;
  const T s1 = S - G / gs;
  const T up = s1 * p[0], vp = s1 * p[1];
  px[0] = up + k[2] * vp + k[3];
  px[1] = k[8] * up + k[1] * vp + k[4];
  return true;
}

inline int scaramuzza_camera_num_params(int model) { return model == SCARAMUZZA ? 9 : camera_num_params(model); }

template <class T> inline bool scaramuzza_project(int model, const T* k, const T* p, T* px, bool dispatch_fov) {
  return model == SCARAMUZZA ? project_scaramuzza(k, p, px) : project<T>(model, k, p, px, dispatch_fov);
}

}  // namespace icco
