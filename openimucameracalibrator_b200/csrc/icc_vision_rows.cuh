// Both residual rows [J | r] of ONE board-corner observation of the rolling-shutter reprojection functor, evaluated jointly.
//
// Reference: RSReprojectionCostFunctorSplit<6>::operator() (basalt_spline/ceres_calib_split_residuals.h:319-402) under
// ceres::DynamicAutoDiffCostFunction x LieLocalParameterization; here the Jacobian is closed form (derivation: header of
// icc_device_math.cuh).  Kept __host__ __device__ so that tests/test_host_device_math.py can compile exactly this code for the
// CPU and check it against finite differences; the persistent vision items (icc_vision_tmem.cu) inlines it unchanged.
//
// What is new against the per-row recursion of icc_spline_chain.cuh (still used by the IMU kernels):
//  * the x and the y row run through the SO(3) knot recursion TOGETHER (two independent dependency chains per lane, shared
//    window loads and shared per-increment coefficients);
//  * the increment rotations are applied in Rodrigues form about the staged unit axis, re-using the two cross products the
//    lambda Jr(lambda d) row product needs anyway (no quaternion sandwich per row);
//  * exp(lambda_i d_i) needs sin/cos of half angles that are < pi/4 for any sane knot spacing: polynomial kernels without
//    range reduction (library sincos beyond that);
//  * only the per-increment (sin, cos) pair is kept (the unit axis is per frame), not the quaternions.
#pragma once
#include <cstddef>
#include "icc_camera.cuh"
#include "icc_bearing_math.cuh"

namespace icc {

// Per-frame quantities, staged once per frame (shared memory in the kernel).
struct FrameWin {
  Q4 q0;                  // first knot of the SO(3) window
  V3 d[5];                // log increments d_i = log(R_i^-1 R_{i+1})
  V3 dh[5];               // unit axes (0 when the increment vanishes)
  double th[5], ith[5];   // |d_i| and its reciprocal (0 when the increment vanishes)
  M3 jri[5];              // Jr^-1(d_i)
  V3 p[6];                // R^3 window
  double u_so3, u_r3;     // normalised knot times of the frame (CalcTimes, impl.h:763-788)
};
struct VisConst {
  double intr[MAX_INTR];
  M3 Ric;                 // rotation matrix of T_i_c
  V3 tic;
  double ld;              // line delay
  int model, fov;
};

// Layout of the parked y row (36 doubles; the R^3 block is kept factored as m_t and the six basis coefficients).
enum { YR_SO3 = 0, YR_MT = 18, YR_DP = 21, YR_OM = 24, YR_LD = 27, YR_R = 28, YR_CC = 29, YR_N = 36 };
// Tile columns of a vision row: [so3 0..17 | r3 18..35 | T_i_c 36..41 | line delay 42 | residual 43]
constexpr int VIS_RES_COL = 43;

// sin / cos for |x| <= pi/4 by the fdlibm kernel polynomials (< 1 ulp there); library sincos beyond.
ICC_HD void sincos_small(double x, double* s, double* c) {
  if (fabs(x) <= 0.78539816339744828) {
    const double z = x * x;
    const double ps = -1.66666666666666324348e-01 + z * (8.33333333332248946124e-03 + z * (-1.98412698298579493134e-04 + z * (2.75573137070700676789e-06 + z * (-2.50507602534068634195e-08 + z * 1.58969099521155010221e-10))));
    const double pc = 4.16666666666666019037e-02 + z * (-1.38888888888741095749e-03 + z * (2.48015872894767294178e-05 + z * (-2.75573143513906633035e-07 + z * (2.08757232129817482790e-09 + z * -1.13596475577881948265e-11))));
    *s = fma(x * z, ps, x);
    *c = fma(z * z, pc, fma(-0.5, z, 1.0));
  } else {
    sincos(x, s, c);
  }
}

// MODEL of the local tangent reprojection error (ICC_REPROJ_ERROR_TANGENT): the corner is its unit bearing b, no camera model is evaluated.
constexpr int VIS_TANGENT = -2;

// One corner.  xrow: entry c of the x row is written to xrow[c * ldx] (c = 0..43).  yr: entry j of the y row in the parked layout
// is written to yr[j * ldy] as soon as it is known, so that the kernel can send it straight to its shared-memory park instead of
// holding the whole row in registers until the end of the corner.
// Failed projection (quirk q12): both residuals are the constant 1e10 with zero Jacobian rows.
// MODEL == VIS_TANGENT: the residual is tangent_projection of the corner's bearing b4 (b_ok: it could be formed) scaled by s, and ox is not
// used; a corner without a bearing is a zero residual with zero rows, one predicted 90 degrees or more off its ray fails as above.
template <int MODEL>   // MODEL >= 0: that camera model only; -1: runtime dispatch on K.model (host tests); VIS_TANGENT: bearings
ICC_HD void vision_corner_rows(const FrameWin& W, const VisConst& K, V3 X, double ox, double oy, double4 b4, bool b_ok, double s, double* __restrict__ xrow, int ldx, double* __restrict__ yr, int ldy, double& r0, double& r1) {
  const double us = W.u_so3 + oy * K.ld, ur = W.u_r3 + oy * K.ld;   // residuals.h:344-346: row time added to the normalised u
  double sn[5], cs[5];
  Q4 q = W.q0;
  {
    double lam[5], dlam[5];
    cum_coeffs6(us, lam, dlam);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      sincos_small(0.5 * lam[i] * W.th[i], &sn[i], &cs[i]);
      const V3 ax = W.dh[i];
      q = qmul(q, q4(sn[i] * ax.x, sn[i] * ax.y, sn[i] * ax.z, cs[i]));
    }
  }
  double cc[6], dc[6];
  coeffs6(ur, cc, dc, nullptr);
  V3 t = v3(0, 0, 0), tdot = v3(0, 0, 0);
#pragma unroll
  for (int j = 0; j < 6; ++j) { t = fma3(cc[j], W.p[j], t); tdot = fma3(dc[j], W.p[j], tdot); }
  const M3 R = qmat(q);                       // R_w_i
  const V3 qi = mulT(R, X - t);               // point in the IMU frame
  const V3 pc = mulT(K.Ric, qi - K.tic);      // point in the camera frame
  Proj pr;
  if constexpr (MODEL == VIS_TANGENT) pr = tangent_projection(b4, b_ok, s, pc);
  else pr = MODEL >= 0 ? project_model<(MODEL >= 0 ? MODEL : 0)>(K.intr, pc, K.fov != 0) : project(K.model, K.intr, pc, K.fov != 0);
  if (!pr.ok) {
    r0 = 1e10; r1 = 1e10;                     // residuals.h:391-393
    if constexpr (MODEL == VIS_TANGENT) { if (!b_ok) { r0 = 0.0; r1 = 0.0; } }
#pragma unroll
    for (int c = 0; c < VIS_RES_COL; ++c) xrow[c * ldx] = 0.0;
    xrow[VIS_RES_COL * ldx] = r0;
#pragma unroll
    for (int c = 0; c < YR_N; ++c) yr[c * ldy] = c == YR_R ? r1 : 0.0;
    return;
  }
  if constexpr (MODEL == VIS_TANGENT) { r0 = pr.u; r1 = pr.v; }
  else { r0 = pr.u - ox; r1 = pr.v - oy; }    // residuals.h:395-398, cov = I
  // Everything but the SO(3) knot columns and the line delay is written before the knot recursion, so that the point, the
  // projection Jacobian and the R^3 coefficients are dead while it runs.
  V3 w[2], zn[2];
  double du[2], mtd[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const V3 Dp = v3(pr.J[3 * r], pr.J[3 * r + 1], pr.J[3 * r + 2]);
    const V3 mq = mul(K.Ric, Dp);             // Dp R_ic^T as a covector
    w[r] = cross(mq, qi);                     // d r / d theta (right increment of R_w_i)
    const V3 mt = mul(R, mq);                 // covector of the translation
    zn[r] = v3(0, 0, 0); du[r] = 0.0;
    mtd[r] = dot(mt, tdot);
    const V3 om = cross(Dp, pc);
    if (r == 0) {
#pragma unroll
      for (int j = 0; j < 6; ++j) { xrow[(18 + 3 * j + 0) * ldx] = -cc[j] * mt.x; xrow[(18 + 3 * j + 1) * ldx] = -cc[j] * mt.y; xrow[(18 + 3 * j + 2) * ldx] = -cc[j] * mt.z; }
      xrow[36 * ldx] = -Dp.x; xrow[37 * ldx] = -Dp.y; xrow[38 * ldx] = -Dp.z;
      xrow[39 * ldx] = om.x; xrow[40 * ldx] = om.y; xrow[41 * ldx] = om.z;
      xrow[VIS_RES_COL * ldx] = r0;
    } else {
#pragma unroll
      for (int j = 0; j < 6; ++j) yr[(YR_CC + j) * ldy] = cc[j];
      yr[YR_MT * ldy] = mt.x; yr[(YR_MT + 1) * ldy] = mt.y; yr[(YR_MT + 2) * ldy] = mt.z;
      yr[YR_DP * ldy] = Dp.x; yr[(YR_DP + 1) * ldy] = Dp.y; yr[(YR_DP + 2) * ldy] = Dp.z;
      yr[YR_OM * ldy] = om.x; yr[(YR_OM + 1) * ldy] = om.y; yr[(YR_OM + 2) * ldy] = om.z;
      yr[YR_R * ldy] = r1;
      yr[(YR_N - 1) * ldy] = 0.0;
    }
  }
  // lambda and its derivative again rather than kept through the projection: ten doubles fewer at the kernel's register peak (the
  // persistent kernel holds its tensor-core accumulators next to this chain).  The empty asm keeps the compiler from merging the two
  // evaluations back into one; the values are the same bits.
  double us_again = us;
#ifdef __CUDA_ARCH__
  asm volatile("" : "+d"(us_again));
#endif
  double lam[5], dlam[5];
  cum_coeffs6(us_again, lam, dlam);
#pragma unroll
  for (int i = 4; i >= 0; --i) {              // increment i couples knots i and i+1
    const double sphi = 2.0 * sn[i] * cs[i], omc = 2.0 * sn[i] * sn[i];          // sin(phi), 1 - cos(phi), phi = lambda_i theta_i
    const double c1 = omc * W.ith[i], c2 = lam[i] - sphi * W.ith[i];              // lambda Jr(lambda d) = lambda I - c1 [dh]x + c2 [dh]x^2
    const V3 dh = W.dh[i], d = W.d[i];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const V3 xd = cross(w[r], dh), xdd = cross(xd, dh);
      const V3 z = v3(lam[i] * w[r].x - c1 * xd.x + c2 * xdd.x, lam[i] * w[r].y - c1 * xd.y + c2 * xdd.y, lam[i] * w[r].z - c1 * xd.z + c2 * xdd.z);
      du[r] = fma(dlam[i], dot(w[r], d), du[r]);
      const V3 up = mulT(W.jri[i], z) - zn[r];          // knot i+1:  z Jr^-1(d_i)  minus what increment i+1 left behind
      zn[r] = mul(W.jri[i], z);                         // knot i:   -Jr^-1(d_i) z  (= -z Jl^-1)
      w[r] = v3(w[r].x - sphi * xd.x + omc * xdd.x, w[r].y - sphi * xd.y + omc * xdd.y, w[r].z - sphi * xd.z + omc * xdd.z);   // exp(lambda d) w
      if (r == 0) { xrow[(3 * (i + 1) + 0) * ldx] = up.x; xrow[(3 * (i + 1) + 1) * ldx] = up.y; xrow[(3 * (i + 1) + 2) * ldx] = up.z; }
      else { yr[(YR_SO3 + 3 * (i + 1) + 0) * ldy] = up.x; yr[(YR_SO3 + 3 * (i + 1) + 1) * ldy] = up.y; yr[(YR_SO3 + 3 * (i + 1) + 2) * ldy] = up.z; }
    }
  }
  {
    const V3 k0 = w[0] - zn[0], k1 = w[1] - zn[1];
    xrow[0] = k0.x; xrow[ldx] = k0.y; xrow[2 * ldx] = k0.z;
    yr[(YR_SO3 + 0) * ldy] = k1.x; yr[(YR_SO3 + 1) * ldy] = k1.y; yr[(YR_SO3 + 2) * ldy] = k1.z;
  }
  xrow[42 * ldx] = oy * (du[0] - mtd[0]);
  yr[YR_LD * ldy] = oy * (du[1] - mtd[1]);
}
template <int MODEL>
ICC_HD void vision_corner_rows(const FrameWin& W, const VisConst& K, V3 X, double ox, double oy, double* __restrict__ xrow, int ldx, double* __restrict__ yr, int ldy, double& r0, double& r1) {
  vision_corner_rows<MODEL>(W, K, X, ox, oy, make_double4(0.0, 0.0, 0.0, 0.0), false, 0.0, xrow, ldx, yr, ldy, r0, r1);
}
template <int MODEL>
ICC_HD void vision_corner_rows(const FrameWin& W, const VisConst& K, V3 X, double ox, double oy, double* __restrict__ xrow, int ldx, double (&yr)[YR_N], double& r0, double& r1) {
  vision_corner_rows<MODEL>(W, K, X, ox, oy, xrow, ldx, yr, 1, r0, r1);
}
template <int MODEL>
ICC_HD void vision_corner_rows(const FrameWin& W, const VisConst& K, V3 X, double oy, double4 b4, bool b_ok, double s, double* __restrict__ xrow, int ldx, double (&yr)[YR_N], double& r0, double& r1) {
  vision_corner_rows<MODEL>(W, K, X, 0.0, oy, b4, b_ok, s, xrow, ldx, yr, 1, r0, r1);
}

// Expand a parked y row into tile entries (what the kernel does after the x rows have been consumed); also used by the CPU test.
ICC_HD void vision_yrow_expand(const double (&yr)[YR_N], double* __restrict__ yrow, int ldy) {
#pragma unroll
  for (int c = 0; c < 18; ++c) yrow[c * ldy] = yr[YR_SO3 + c];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    yrow[(18 + 3 * j + 0) * ldy] = -yr[YR_CC + j] * yr[YR_MT]; yrow[(18 + 3 * j + 1) * ldy] = -yr[YR_CC + j] * yr[YR_MT + 1]; yrow[(18 + 3 * j + 2) * ldy] = -yr[YR_CC + j] * yr[YR_MT + 2];
  }
  yrow[36 * ldy] = -yr[YR_DP]; yrow[37 * ldy] = -yr[YR_DP + 1]; yrow[38 * ldy] = -yr[YR_DP + 2];
  yrow[39 * ldy] = yr[YR_OM]; yrow[40 * ldy] = yr[YR_OM + 1]; yrow[41 * ldy] = yr[YR_OM + 2];
  yrow[42 * ldy] = yr[YR_LD];
  yrow[VIS_RES_COL * ldy] = yr[YR_R];
}

// The increment between two SO(3) knots: d = log(qa^-1 qb), |d| and its reciprocal (0 when the increment vanishes), the unit axis
// and Jr^-1(d).  The one copy of this code: the window staging below and the increment table both call it.
ICC_HD void so3_increment(Q4 qa, Q4 qb, V3& d_out, V3& dh, double& th_out, double& ith_out, M3& jri) {
  const V3 d = so3_log(qmul(qconj(qa), qb));
  d_out = d;
  const double th = sqrt(dot(d, d)), ith = th > 1e-150 ? 1.0 / th : 0.0;
  th_out = th; ith_out = ith; dh = ith * d;
  jri = so3_jr_inv(d);
}

// Window staging for one frame from its six SO(3) knots (x,y,z,w) and six R^3 knots; `i` < 5 handles increment i.
ICC_HD void stage_frame_increment(FrameWin& W, int i, Q4 qa, Q4 qb) { so3_increment(qa, qb, W.d[i], W.dh[i], W.th[i], W.ith[i], W.jri[i]); }

// ---- SO(3) increment table ----------------------------------------------------------------------------------------------------
// Entry i < n (= n_so3 - 1) is the increment between knots i and i + 1 of one state (so3_increment), formed once per evaluation by
// incr_table_kernel (icc_eval_tmem.cu) instead of once per staged window.  It is stored field by field -- d (3n doubles), dh (3n),
// th (n), ith (n), jri (9n) -- so that the five increments of the window that starts at knot s are five contiguous runs in FrameWin's
// own order from FrameWin::d to FrameWin::jri: staging a window's increments is an 85-double copy.
constexpr int INCR_DOUBLES = 17;                      // doubles per entry
constexpr int WIN_INCR_DOUBLES = 5 * INCR_DOUBLES;    // FrameWin::d .. FrameWin::jri
static_assert(offsetof(FrameWin, dh) == offsetof(FrameWin, d) + 15 * sizeof(double) && offsetof(FrameWin, th) == offsetof(FrameWin, d) + 30 * sizeof(double) &&
              offsetof(FrameWin, ith) == offsetof(FrameWin, d) + 35 * sizeof(double) && offsetof(FrameWin, jri) == offsetof(FrameWin, d) + 40 * sizeof(double) &&
              offsetof(FrameWin, p) == offsetof(FrameWin, d) + WIN_INCR_DOUBLES * sizeof(double), "FrameWin's increment block: d, dh, th, ith, jri back to back");

ICC_HD void incr_table_entry(const double4* __restrict__ so3, int i, int n, double* __restrict__ tab) {
  const double4 a = so3[i], b = so3[i + 1];
  V3 d, dh; double th, ith; M3 jri;
  so3_increment(q4(a.x, a.y, a.z, a.w), q4(b.x, b.y, b.z, b.w), d, dh, th, ith, jri);
  tab[3 * i] = d.x; tab[3 * i + 1] = d.y; tab[3 * i + 2] = d.z;
  tab[3 * n + 3 * i] = dh.x; tab[3 * n + 3 * i + 1] = dh.y; tab[3 * n + 3 * i + 2] = dh.z;
  tab[6 * n + i] = th; tab[7 * n + i] = ith;
#pragma unroll
  for (int k = 0; k < 9; ++k) tab[8 * n + 9 * i + k] = jri.m[k];
}
// Table index of double e (< WIN_INCR_DOUBLES) of the increment block of the window that starts at knot s.
ICC_HD int incr_table_index(int e, int s, int n) {
  if (e < 15) return 3 * s + e;
  if (e < 30) return 3 * n + 3 * s + (e - 15);
  if (e < 35) return 6 * n + s + (e - 30);
  if (e < 40) return 7 * n + s + (e - 35);
  return 8 * n + 9 * s + (e - 40);
}
ICC_HD double* win_incr(FrameWin& W) { return &W.d[0].x; }

}  // namespace icc
