// The CPU oracle with SCARAMUZZA (Scaramuzza's omnidirectional polynomial model, model id 8), for tests/test_scaramuzza.py and
// tests/test_gpu_scaramuzza.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more, unchanged, into a library of its own (by default through
// tests/rolling_shutter/rs_camcal_oracle.cpp, so that the library also has the rolling-shutter camera calibration; with -DSCARAMUZZA_TANGENT
// through tests/tangent_spline/tangent_oracle.cpp, for the tangent reprojection error), with the substitutions of
// tests/omni_radtan/omni_oracle.cpp:
//   * every `project<T>(` and `camera_num_params(` of the oracle resolves to scaramuzza_project / scaramuzza_camera_num_params
//     (scaramuzza_oracle_math.hpp), which add the model and hand every other model to the oracle's own functions;
//   * every call `camcal_bundle_adjust(C, ...)` of the camera calibration resolves to scaramuzza_camcal_bundle_adjust below, and the
//     definition `camcal_bundle_adjust(CamCal& C, ...)` is renamed camcal_bundle_adjust_oracle (the macro pastes the first argument's first
//     token, `C` at the calls and `CamCal` at the definition).  scaramuzza_camcal_bundle_adjust gives model 8 the schedule of the product's
//     calibration (icc_camcal.cu): the radial subset {a2, a3, a4} in stage 1, starting from the stereographic member a2 = -1 / (4 a0);
//     the stretch {e, d} in stage 3.  Every other model (and the division-model initialiser) runs the oracle's bundle adjustment unchanged.
// Everything else is the oracle's own code.
#include "scaramuzza_oracle_math.hpp"
#include "../../include/icc_b200.h"

namespace {
struct CamCal;
struct CamCalStage;
CamCalStage scaramuzza_camcal_bundle_adjust(CamCal& C, unsigned mask, bool pose_free, const icc_camcal_options& o);
}  // namespace

#define project scaramuzza_project
#define camera_num_params scaramuzza_camera_num_params
#define camcal_bundle_adjust(first, ...) SCARA_CCBA_##first, __VA_ARGS__)
#define SCARA_CCBA_C scaramuzza_camcal_bundle_adjust(C
#define SCARA_CCBA_CamCal camcal_bundle_adjust_oracle(CamCal
#ifdef SCARAMUZZA_TANGENT
#include "../tangent_spline/tangent_oracle.cpp"
#else
#include "../rolling_shutter/rs_camcal_oracle.cpp"
#endif
#undef project
#undef camera_num_params
#undef camcal_bundle_adjust
#undef SCARA_CCBA_C
#undef SCARA_CCBA_CamCal

namespace {
CamCalStage scaramuzza_camcal_bundle_adjust(CamCal& C, unsigned mask, bool pose_free, const icc_camcal_options& o) {
  if (C.model == SCARAMUZZA) {
    if (mask & (1u << 5)) {                          // stage 1: a0 + the oracle's default radial subset {5, 6}
      mask |= 1u << 7;
      C.k[5] = -0.25 / C.k[0];                       // the stereographic member: magnification a0 = f0 at the image centre
    } else if (pose_free) {                          // stage 3 (and its repeat after the board-point refinement)
      mask |= (1u << 2) | (1u << 8);
    }
  }
  return camcal_bundle_adjust_oracle(C, mask, pose_free, o);
}
}  // namespace
