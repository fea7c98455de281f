// OMNI_RADIAL_TANGENTIAL (Kalibr's omni-radtan, model id 7) for the CPU oracle, test infrastructure only.  oracle/oracle_math.hpp states the
// reference's camera models and stays as it is; this header states the extension model from its published equations in the same templated
// form, so that the oracle's Jet autodiff differentiates it, and dispatches to the oracle's own `project` for every other model.
#pragma once
#include "../../oracle/oracle_math.hpp"

namespace icco {

constexpr int OMNI_RADIAL_TANGENTIAL = 7;

// [f, ar, skew, cx, cy, xi, k1, k2, t1, t2]: n = z + xi |p|, (x, y) / n distorted radially (k1, k2) and tangentially (t1, t2), skewed affine;
// valid iff z > -w |p|, w = xi <= 1 ? xi : 1 / xi
template <class T> inline bool project_omni_radial_tangential(const T* k, const T* p, T* px) {
  const T xi = k[5];
  const T d = jsqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
  const T w = xi <= 1.0 ? xi : 1.0 / xi;
  if (p[2] <= -w * d) return false;
  const T n = p[2] + xi * d;
  const T x = p[0] / n, y = p[1] / n;
  const T r2 = x * x + y * y;
  const T radial = 1.0 + k[6] * r2 + k[7] * r2 * r2;
  const T dx = x * radial + 2.0 * k[8] * x * y + k[9] * (r2 + 2.0 * x * x);
  const T dy = y * radial + 2.0 * k[9] * x * y + k[8] * (r2 + 2.0 * y * y);
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}

inline int omni_camera_num_params(int model) { return model == OMNI_RADIAL_TANGENTIAL ? 10 : camera_num_params(model); }

template <class T> inline bool omni_project(int model, const T* k, const T* p, T* px, bool dispatch_fov) {
  return model == OMNI_RADIAL_TANGENTIAL ? project_omni_radial_tangential(k, p, px) : project<T>(model, k, p, px, dispatch_fov);
}

}  // namespace icco
