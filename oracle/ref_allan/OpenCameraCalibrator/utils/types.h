// Stand-in for the reference's OpenCameraCalibrator/utils/types.h: the two value classes its Allan variance code uses, nothing else.
#pragma once
#include <string>
namespace OpenICC {
struct AccData { double a = 0.0, t = 0.0; AccData() = default; AccData(double d, double time) : a(d), t(time) {} };
struct GyrData { double w = 0.0, t = 0.0; GyrData() = default; GyrData(double d, double time) : w(d), t(time) {} };
}  // namespace OpenICC
