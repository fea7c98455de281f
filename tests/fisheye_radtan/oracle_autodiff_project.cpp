// The oracle-form FISHEYE_RADIAL_TANGENTIAL projection (fisheye_radtan_oracle_math.hpp) on the oracle's dual numbers, so that
// tests/test_fisheye_radtan.py can hold the product's closed-form Jacobians against autodiff.  Test infrastructure only.
#include "fisheye_radtan_oracle_math.hpp"

using namespace icco;

extern "C" {
// px[2], Jp[2x3] = d px / d point, Jk[2x13] = d px / d intrinsics (row-major)
void oad_fisheye_radtan_project(const double* k, const double* p, double* px, double* Jp, double* Jk) {
  typedef Jet<3 + FISHEYE_RADTAN_N> J;
  J kk[FISHEYE_RADTAN_N], pp[3], out[2];
  for (int i = 0; i < FISHEYE_RADTAN_N; ++i) { kk[i] = J(k[i]); kk[i].v[3 + i] = 1.0; }
  for (int i = 0; i < 3; ++i) { pp[i] = J(p[i]); pp[i].v[i] = 1.0; }
  fisheye_radtan_project<J>(kk, pp, out);
  for (int r = 0; r < 2; ++r) {
    px[r] = out[r].a;
    for (int j = 0; j < 3; ++j) Jp[3 * r + j] = out[r].v[j];
    for (int q = 0; q < FISHEYE_RADTAN_N; ++q) Jk[FISHEYE_RADTAN_N * r + q] = out[r].v[3 + q];
  }
}
}
