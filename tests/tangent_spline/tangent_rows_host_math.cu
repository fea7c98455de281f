// The spline solve's tangent reprojection rows (icc_vision_rows.cuh, MODEL = VIS_TANGENT) and its pixel scale compiled for the CPU, so that
// tests/test_tangent_spline.py can check every Jacobian column against central differences of the same residual.
#include "../../openimucameracalibrator_b200/csrc/icc_vision_rows.cuh"

using namespace icc;

namespace {
void stage(FrameWin& W, VisConst& K, const double* so3, const double* r3, double u_so3, double u_r3, const double* T_ic, double ld) {
  for (int i = 0; i < 5; ++i) stage_frame_increment(W, i, q4(so3[4 * i], so3[4 * i + 1], so3[4 * i + 2], so3[4 * i + 3]), q4(so3[4 * i + 4], so3[4 * i + 5], so3[4 * i + 6], so3[4 * i + 7]));
  W.q0 = q4(so3[0], so3[1], so3[2], so3[3]); W.u_so3 = u_so3; W.u_r3 = u_r3;
  for (int j = 0; j < 6; ++j) W.p[j] = v3(r3[3 * j], r3[3 * j + 1], r3[3 * j + 2]);
  for (int i = 0; i < 10; ++i) K.intr[i] = 0.0;
  K.Ric = qmat(q4(T_ic[0], T_ic[1], T_ic[2], T_ic[3])); K.tic = v3(T_ic[4], T_ic[5], T_ic[6]); K.ld = ld; K.model = -1; K.fov = 0;
}
}  // namespace

extern "C" {
// Both rows [J | r] (2 x 44, row-major) of one corner with bearing b (ok: it exists) and scale s.  so3 = 6 x (x,y,z,w), r3 = 6 x 3,
// T_ic = (qx,qy,qz,qw,tx,ty,tz).  Returns 1 when the residual is defined, 0 for the 1e10 constant, -1 for a corner without a bearing.
int ts_tangent_rows(const double* so3, const double* r3, double u_so3, double u_r3, const double* T_ic, double ld, const double* X, double oy,
                    const double* b, int ok, double s, double* rows) {
  static FrameWin W; VisConst K;
  stage(W, K, so3, r3, u_so3, u_r3, T_ic, ld);
  double yr[YR_N], r0, r1;
  vision_corner_rows<VIS_TANGENT>(W, K, v3(X[0], X[1], X[2]), oy, make_double4(b[0], b[1], b[2], 0.0), ok != 0, s, rows, 1, yr, r0, r1);
  vision_yrow_expand(yr, rows + 44, 1);
  return r0 == 1e10 ? 0 : (ok ? 1 : -1);
}
// The same corner through the pixel rows of a camera model (pixel (ox, oy)); returns 0 when the projection fails.
int ts_pixel_rows(int model, const double* intr10, const double* so3, const double* r3, double u_so3, double u_r3, const double* T_ic, double ld,
                  const double* X, double ox, double oy, double* rows) {
  static FrameWin W; VisConst K;
  stage(W, K, so3, r3, u_so3, u_r3, T_ic, ld);
  for (int i = 0; i < 10; ++i) K.intr[i] = intr10[i];
  K.model = model; K.fov = 1;
  double yr[YR_N], r0, r1;
  vision_corner_rows<-1>(W, K, v3(X[0], X[1], X[2]), ox, oy, rows, 1, yr, r0, r1);
  vision_yrow_expand(yr, rows + 44, 1);
  return r0 == 1e10 ? 0 : 1;
}
double ts_tangent_scale(int model, const double* intr10, int fov) { return tangent_scale(model, intr10, fov != 0); }
}
