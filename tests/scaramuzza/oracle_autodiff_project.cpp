// The oracle's templated camera projection (oracle/oracle_math.hpp, with SCARAMUZZA from scaramuzza_oracle_math.hpp) evaluated on dual
// numbers, so that tests/test_scaramuzza.py can hold the product's implicit-function Jacobians against autodiff.  Test infrastructure only.
#include "scaramuzza_oracle_math.hpp"

using namespace icco;

extern "C" {
// px[2], Jp[2x3] = d px / d point, Jk[2x10] = d px / d intrinsics (row-major); returns the model's domain verdict
int oad_project(int model, const double* k, const double* p, double* px, double* Jp, double* Jk) {
  typedef Jet<13> J;
  J kk[10], pp[3], out[2];
  for (int i = 0; i < 10; ++i) { kk[i] = J(k[i]); kk[i].v[3 + i] = 1.0; }
  for (int i = 0; i < 3; ++i) { pp[i] = J(p[i]); pp[i].v[i] = 1.0; }
  const bool ok = scaramuzza_project<J>(model, kk, pp, out, true);
  for (int r = 0; r < 2; ++r) {
    px[r] = out[r].a;
    for (int j = 0; j < 3; ++j) Jp[3 * r + j] = out[r].v[j];
    for (int q = 0; q < 10; ++q) Jk[10 * r + q] = out[r].v[3 + q];
  }
  return ok ? 1 : 0;
}
}
