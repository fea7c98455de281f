// The CPU oracle with OMNI_RADIAL_TANGENTIAL (Kalibr's omni-radtan, model id 7), for tests/test_omni_radtan.py and
// tests/test_gpu_omni_radtan.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more, unchanged, into a library of its own (by default through
// tests/rolling_shutter/rs_camcal_oracle.cpp, so that the library also has the rolling-shutter camera calibration; with -DOMNI_TANGENT through
// tests/tangent_spline/tangent_oracle.cpp, for the tangent reprojection error), with three substitutions:
//   * every `project<T>(` and `camera_num_params(` of the oracle resolves to omni_project / omni_camera_num_params (omni_oracle_math.hpp),
//     which add the model and hand every other model to the oracle's own functions;
//   * every call `camcal_bundle_adjust(C, ...)` of the camera calibration resolves to omni_camcal_bundle_adjust below, and the definition
//     `camcal_bundle_adjust(CamCal& C, ...)` is renamed camcal_bundle_adjust_oracle: the function-like macro pastes its first argument's first
//     token, `C` at the calls and `CamCal` at the definition, onto OMNI_CCBA_ and so tells the two apart.
//     omni_camcal_bundle_adjust gives model 7 the schedule of the product's calibration (icc_camcal.cu): the radial subset {xi, k1, k2} in
//     stage 1, starting from xi = 1 and f = 2 f0; the tangential subset {t1, t2} in stage 3.  Every other model (and the division-model
//     initialiser) runs the oracle's bundle adjustment unchanged.
// Everything else is the oracle's own code.
#include "omni_oracle_math.hpp"
#include "../../include/icc_b200.h"

namespace {
struct CamCal;
struct CamCalStage;
CamCalStage omni_camcal_bundle_adjust(CamCal& C, unsigned mask, bool pose_free, const icc_camcal_options& o);
}  // namespace

#define project omni_project
#define camera_num_params omni_camera_num_params
#define camcal_bundle_adjust(first, ...) OMNI_CCBA_##first, __VA_ARGS__)
#define OMNI_CCBA_C omni_camcal_bundle_adjust(C
#define OMNI_CCBA_CamCal camcal_bundle_adjust_oracle(CamCal
#ifdef OMNI_TANGENT
#include "../tangent_spline/tangent_oracle.cpp"
#else
#include "../rolling_shutter/rs_camcal_oracle.cpp"
#endif
#undef project
#undef camera_num_params
#undef camcal_bundle_adjust
#undef OMNI_CCBA_C
#undef OMNI_CCBA_CamCal

namespace {
CamCalStage omni_camcal_bundle_adjust(CamCal& C, unsigned mask, bool pose_free, const icc_camcal_options& o) {
  if (C.model == OMNI_RADIAL_TANGENTIAL) {
    if (mask & (1u << 5)) {                          // stage 1: focal length + the oracle's default radial subset {5, 6}
      mask |= 1u << 7;
      C.k[5] = 1.0; C.k[0] *= 2.0;                   // xi = 1, f = (1 + xi) f0: magnification f0 at the image centre
    } else if (pose_free) {                          // stage 3 (and its repeat after the board-point refinement)
      mask |= (1u << 8) | (1u << 9);
    }
  }
  return camcal_bundle_adjust_oracle(C, mask, pose_free, o);
}
}  // namespace
