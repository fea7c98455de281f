// The CPU oracle with PINHOLE_RATIONAL (OpenCV's rational polynomial model, model id 9) for the spline evaluation and LM, for
// tests/test_gpu_rational.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more, unchanged, into a library of its own (with -DRATIONAL_TANGENT
// through tests/tangent_spline/tangent_oracle.cpp, for the tangent reprojection error), with the substitution of
// tests/omni_radtan/omni_oracle.cpp: every `project<T>(` and `camera_num_params(` of the oracle resolves to rational_oracle_project_any /
// rational_camera_num_params below, which add the model and hand every other model to the oracle's own functions.  The oracle holds ten
// intrinsics per camera, so it sees model 9 with ten parameters and keeps the denominator k4, k5, k6 constant
// (rational_oracle_set_denominator): its CAM_INTRINSICS columns are the first ten of the product's thirteen.
#include "rational_oracle_math.hpp"

namespace icco {
inline int rational_camera_num_params(int model) { return model == PINHOLE_RATIONAL ? 10 : camera_num_params(model); }
template <class T> inline bool rational_oracle_project_any(int model, const T* k, const T* p, T* px, bool dispatch_fov) {
  return model == PINHOLE_RATIONAL ? rational_oracle_project(k, p, px) : project<T>(model, k, p, px, dispatch_fov);
}
}  // namespace icco

#define project rational_oracle_project_any
#define camera_num_params rational_camera_num_params
#ifdef RATIONAL_TANGENT
#include "../tangent_spline/tangent_oracle.cpp"
#else
#include "../../oracle/icc_oracle.cpp"
#endif
#undef project
#undef camera_num_params

extern "C" void rational_oracle_set_denominator(const double* k456) { for (int i = 0; i < 3; ++i) icco::g_rational_den[i] = k456[i]; }
