// The CPU oracle with FISHEYE_RADIAL_TANGENTIAL (Kannala-Brandt with six radial and two tangential terms, model id 10) for the spline
// evaluation and LM, for tests/test_gpu_fisheye_radtan.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more, unchanged, into a library of its own (with
// -DFISHEYE_RADTAN_TANGENT through tests/tangent_spline/tangent_oracle.cpp, for the tangent reprojection error), with the substitution of
// tests/rational/rational_oracle.cpp: every `project<T>(` and `camera_num_params(` of the oracle resolves to fisheye_radtan_oracle_project_any
// / fisheye_radtan_camera_num_params below, which add the model and hand every other model to the oracle's own functions.  The oracle holds
// ten intrinsics per camera, so it sees model 10 with ten parameters ([f, ar, skew, cx, cy, k1..k5]) and keeps k6, t1, t2 constant
// (fisheye_radtan_oracle_set_tail): its CAM_INTRINSICS columns are the first ten of the product's thirteen.
#include "fisheye_radtan_oracle_math.hpp"

namespace icco {
inline double g_fisheye_radtan_tail[3] = {0.0, 0.0, 0.0};   // k6, t1, t2

template <class T> inline double fr_scalar(const T& v) { return v.a; }
inline double fr_scalar(double v) { return v; }

template <class T> inline bool fisheye_radtan_oracle_project(const T* k10, const T* p, T* px) {
  T k[FISHEYE_RADTAN_N];
  for (int i = 0; i < 10; ++i) k[i] = k10[i];
  for (int i = 0; i < 3; ++i) k[10 + i] = T(g_fisheye_radtan_tail[i]);
  double kd[FISHEYE_RADTAN_N];
  for (int i = 0; i < FISHEYE_RADTAN_N; ++i) kd[i] = fr_scalar(k[i]);
  if (!fisheye_radtan_oracle_in_domain(kd, fr_scalar(p[0]), fr_scalar(p[1]), fr_scalar(p[2]))) { px[0] = T(0.0); px[1] = T(0.0); return false; }
  fisheye_radtan_project<T>(k, p, px);
  return true;
}

inline int fisheye_radtan_camera_num_params(int model) { return model == FISHEYE_RADIAL_TANGENTIAL ? 10 : camera_num_params(model); }
template <class T> inline bool fisheye_radtan_oracle_project_any(int model, const T* k, const T* p, T* px, bool dispatch_fov) {
  return model == FISHEYE_RADIAL_TANGENTIAL ? fisheye_radtan_oracle_project(k, p, px) : project<T>(model, k, p, px, dispatch_fov);
}
}  // namespace icco

#define project fisheye_radtan_oracle_project_any
#define camera_num_params fisheye_radtan_camera_num_params
#ifdef FISHEYE_RADTAN_TANGENT
#include "../tangent_spline/tangent_oracle.cpp"
#else
#include "../../oracle/icc_oracle.cpp"
#endif
#undef project
#undef camera_num_params

extern "C" void fisheye_radtan_oracle_set_tail(const double* k6_t1_t2) { for (int i = 0; i < 3; ++i) icco::g_fisheye_radtan_tail[i] = k6_t1_t2[i]; }
