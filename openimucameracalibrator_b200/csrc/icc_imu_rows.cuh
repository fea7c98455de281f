// The three accelerometer rows and the three gyroscope rows [J | r] of ONE IMU sample, each triple evaluated jointly.
//
// Reference: AccelerationCostFunctorSplit<6>::operator() (basalt_spline/ceres_calib_split_residuals.h:52-93) and
// GyroCostFunctorSplit<6,SO3,false>::operator() (:133-169) under ceres::DynamicAutoDiffCostFunction x LieLocalParameterization,
// with the body-velocity recursion of CeresSplineHelper::evaluate_lie (ceres_spline_helper.h:159-164).  Closed-form Jacobians w.r.t.
// right increments of the six SO(3) knots, the six R^3 knots and gravity (the column set of the hot CLI's stage 1 with the biases
// fixed: the wider column sets -- bias knots, IMU intrinsics, time offset -- stay on imu_kernel of icc_eval.cu).
// __host__ __device__ so that tests/test_host_device_math.py can check exactly this code against finite differences on the CPU;
// the persistent IMU items (icc_imu_tmem.cu) inlines it unchanged.
//
// As in icc_vision_rows.cuh: the three rows of a triple share one pass through the knot recursion (three independent dependency
// chains per lane, shared window loads and per-increment coefficients), increment rotations are applied in Rodrigues form about
// the staged unit axes, half-angle sin/cos come from the polynomial kernels, and only (sin, cos) per increment is kept.
#pragma once
#include "icc_vision_rows.cuh"

namespace icc {

struct ImuWin {
  FrameWin f;             // SO(3) increments + R^3 window (u_so3 / u_r3 unused: per sample)
  V3 ba[3], bg[3];        // bias-spline windows
};
struct ImuConst {
  double Ma[9], Mg[9];    // misalignment * scale matrices (utils/types.h:226-246)
  V3 grav;
  double w_acc, w_gyr;    // 1 / std_r3, 1 / std_so3
  double idt2;            // inv_r3_dt^2
  double inv_so3_dt;
  double du_so3, du_r3, du_ba, du_bg;   // time-offset terms of the normalised spline times (persistent kernel only)
};

// Tile columns.  accelerometer: [so3 0..17 | r3 18..35 | gravity 36..38 | residual 39] (5 blocks of 8, no padding);
// gyroscope: [so3 0..17 | residual 18 | zero 19..23] (3 blocks of 8)
constexpr int ACC_RES_COL = 39, GYR_RES_COL = 18;
// parked layouts: accelerometer rows 1, 2 = [so3 row 1 (18) | so3 row 2 (18) | q (4) | r1 | r2 | u_r3] ; gyroscope rows 1, 2 = [row 1 (18) | row 2 (18) | r1 | r2]
constexpr int ACC_PARK = 43, GYR_PARK = 38;

// second u-derivative of the non-cumulative coefficients only
ICC_HD void coeffs6_dd_only(double u, double ddc[6]) {
  const double k = 1.0 / 120.0, u2 = u * u, u3 = u2 * u;
  ddc[0] = k * (20.0 - 60.0 * u + 60.0 * u2 - 20.0 * u3);
  ddc[1] = k * (40.0 + 120.0 * u - 240.0 * u2 + 100.0 * u3);
  ddc[2] = k * (-120.0 + 360.0 * u2 - 200.0 * u3);
  ddc[3] = k * (40.0 - 120.0 * u - 240.0 * u2 + 200.0 * u3);
  ddc[4] = k * (20.0 + 60.0 * u + 60.0 * u2 - 100.0 * u3);
  ddc[5] = k * (20.0 * u3);
}

// accelerometer rows.  row0: entry c at row0[c * ld] (c = 0..39).  pk: entry j of rows 1 and 2 in the parked layout is written to
// pk[j * ldp] as soon as it is known, so that the kernel can send it straight to its shared-memory park instead of holding both rows
// in registers until the end of the sample.  Everything but the SO(3) knot columns is written before the knot recursion, so that R,
// the R^3 coefficients and the quaternion are dead while it runs.
ICC_HD void imu_accel_rows(const ImuWin& W, const ImuConst& K, double u_so3, double u_r3, double u_ba, V3 a_meas, double* __restrict__ row0, int ld, double* __restrict__ pk, int ldp, double (&ra)[3]) {
  const FrameWin& F = W.f;
  double lam[5], dlam[5], sn[5], cs[5];
  cum_coeffs6(u_so3, lam, dlam);
  Q4 q = F.q0;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    sincos_small(0.5 * lam[i] * F.th[i], &sn[i], &cs[i]);
    const V3 ax = F.dh[i];
    q = qmul(q, q4(sn[i] * ax.x, sn[i] * ax.y, sn[i] * ax.z, cs[i]));
  }
  double ddc[6], cba[3];
  coeffs6_dd_only(u_r3, ddc); coeffs3(u_ba, cba);
  V3 aw = v3(0, 0, 0);
#pragma unroll
  for (int j = 0; j < 6; ++j) aw = fma3(ddc[j] * K.idt2, F.p[j], aw);
  const M3 R = qmat(q);
  const V3 h = mulT(R, aw + K.grav);                          // R_w_i^T (p'' + g)   (residuals.h:88)
  V3 bacc = v3(0, 0, 0);
#pragma unroll
  for (int k = 0; k < 3; ++k) bacc = fma3(cba[k], W.ba[k], bacc);
  const V3 a_raw = a_meas - bacc;
  ra[0] = K.w_acc * (h.x - (K.Ma[0] * a_raw.x + K.Ma[1] * a_raw.y + K.Ma[2] * a_raw.z));
  ra[1] = K.w_acc * (h.y - (K.Ma[3] * a_raw.x + K.Ma[4] * a_raw.y + K.Ma[5] * a_raw.z));
  ra[2] = K.w_acc * (h.z - (K.Ma[6] * a_raw.x + K.Ma[7] * a_raw.y + K.Ma[8] * a_raw.z));
  // row 0: R^3 knots, gravity, residual.  m_t = R e_0 = first column of R
  {
    const V3 mt = v3(R.m[0], R.m[3], R.m[6]);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const double s = K.w_acc * ddc[j] * K.idt2;
      row0[(18 + 3 * j + 0) * ld] = s * mt.x; row0[(18 + 3 * j + 1) * ld] = s * mt.y; row0[(18 + 3 * j + 2) * ld] = s * mt.z;
    }
    row0[36 * ld] = K.w_acc * mt.x; row0[37 * ld] = K.w_acc * mt.y; row0[38 * ld] = K.w_acc * mt.z;
    row0[ACC_RES_COL * ld] = ra[0];
  }
  pk[36 * ldp] = q.x; pk[37 * ldp] = q.y; pk[38 * ldp] = q.z; pk[39 * ldp] = q.w;
  pk[40 * ldp] = ra[1]; pk[41 * ldp] = ra[2]; pk[42 * ldp] = u_r3;
  // d r_k / d theta = w_acc (e_k x h)  (row covector, right increment of R_w_i)
  V3 w[3], zn[3];
  // cross(e_0, h) = (0, -h.z, h.y), cross(e_1, h) = (h.z, 0, -h.x), cross(e_2, h) = (-h.y, h.x, 0)
  w[0] = v3(0.0, -K.w_acc * h.z, K.w_acc * h.y);
  w[1] = v3(K.w_acc * h.z, 0.0, -K.w_acc * h.x);
  w[2] = v3(-K.w_acc * h.y, K.w_acc * h.x, 0.0);
#pragma unroll
  for (int r = 0; r < 3; ++r) zn[r] = v3(0, 0, 0);
#pragma unroll
  for (int i = 4; i >= 0; --i) {
    const double sphi = 2.0 * sn[i] * cs[i], omc = 2.0 * sn[i] * sn[i];
    const double c1 = omc * F.ith[i], c2 = lam[i] - sphi * F.ith[i];
    const V3 dh = F.dh[i];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const V3 xd = cross(w[r], dh), xdd = cross(xd, dh);
      const V3 z = v3(lam[i] * w[r].x - c1 * xd.x + c2 * xdd.x, lam[i] * w[r].y - c1 * xd.y + c2 * xdd.y, lam[i] * w[r].z - c1 * xd.z + c2 * xdd.z);
      const V3 up = mulT(F.jri[i], z) - zn[r];
      zn[r] = mul(F.jri[i], z);
      w[r] = v3(w[r].x - sphi * xd.x + omc * xdd.x, w[r].y - sphi * xd.y + omc * xdd.y, w[r].z - sphi * xd.z + omc * xdd.z);
      if (r == 0) { row0[(3 * (i + 1) + 0) * ld] = up.x; row0[(3 * (i + 1) + 1) * ld] = up.y; row0[(3 * (i + 1) + 2) * ld] = up.z; }
      else { pk[(18 * (r - 1) + 3 * (i + 1) + 0) * ldp] = up.x; pk[(18 * (r - 1) + 3 * (i + 1) + 1) * ldp] = up.y; pk[(18 * (r - 1) + 3 * (i + 1) + 2) * ldp] = up.z; }
    }
  }
  {
    const V3 k0 = w[0] - zn[0], k1 = w[1] - zn[1], k2 = w[2] - zn[2];
    row0[0] = k0.x; row0[ld] = k0.y; row0[2 * ld] = k0.z;
    pk[0] = k1.x; pk[ldp] = k1.y; pk[2 * ldp] = k1.z;
    pk[18 * ldp] = k2.x; pk[19 * ldp] = k2.y; pk[20 * ldp] = k2.z;
  }
}
// park: rows 1 and 2 in the parked layout (the CPU test and the host harness)
ICC_HD void imu_accel_rows(const ImuWin& W, const ImuConst& K, double u_so3, double u_r3, double u_ba, V3 a_meas, double* __restrict__ row0, int ld, double (&park)[ACC_PARK], double (&ra)[3]) {
  imu_accel_rows(W, K, u_so3, u_r3, u_ba, a_meas, row0, ld, park, 1, ra);
}

// expand one parked accelerometer row (k = 1 or 2) into tile entries: so3 = its 18 knot entries, then the shared tail of the
// parked layout (quaternion of R_w_i, residual of this row, u_r3).  An all-zero quaternion marks a padding lane: zero row.
ICC_HD void imu_accel_row_expand(const double (&so3)[18], Q4 q, double res, double u_r3, const ImuConst& K, int k, double* __restrict__ row, int ld) {
  const bool live = q.x != 0.0 || q.y != 0.0 || q.z != 0.0 || q.w != 0.0;
#pragma unroll
  for (int c = 0; c < 18; ++c) row[c * ld] = so3[c];
  const M3 R = qmat(q);
  const double wl = live ? K.w_acc : 0.0;
  const V3 mt = k == 1 ? v3(R.m[1], R.m[4], R.m[7]) : v3(R.m[2], R.m[5], R.m[8]);
  double ddc[6];
  coeffs6_dd_only(u_r3, ddc);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const double s = wl * ddc[j] * K.idt2;
    row[(18 + 3 * j + 0) * ld] = s * mt.x; row[(18 + 3 * j + 1) * ld] = s * mt.y; row[(18 + 3 * j + 2) * ld] = s * mt.z;
  }
  row[36 * ld] = wl * mt.x; row[37 * ld] = wl * mt.y; row[38 * ld] = wl * mt.z;
  row[ACC_RES_COL * ld] = res;
}

// gyroscope rows.  row0: entry c at row0[c * ld] (c = 0..23, 19..23 zero).  pk: entry j of rows 1 and 2 in the parked layout at
// pk[j * ldp], written as soon as it is known (the residuals before the knot recursion).
ICC_HD void imu_gyro_rows(const ImuWin& W, const ImuConst& K, double u_so3, double u_bg, V3 g_meas, double* __restrict__ row0, int ld, double* __restrict__ pk, int ldp, double (&rg)[3]) {
  const FrameWin& F = W.f;
  double lam[5], dlam[5], sn[5], cs[5], cbg[3];
  cum_coeffs6(u_so3, lam, dlam);
  coeffs3(u_bg, cbg);
  // body velocity: omega <- A_i^T omega + lambda'_i d_i / dt   (ceres_spline_helper.h:159-164); s_i = A_i^T omega_{i-1}.
  // The Jacobian recursion needs s_i again, in reverse order.  Rather than holding all five through it (15 doubles at the kernel's
  // register peak: the persistent kernel keeps its tensor-core accumulators next to this chain), s_i waits in the parked slots of
  // row 1's knot i+1, which the recursion overwrites only after its last read of s_i.  The volatile read keeps the compiler from
  // forwarding the stored registers; the values are the same bits.
  V3 om = v3(0, 0, 0);
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    sincos_small(0.5 * lam[i] * F.th[i], &sn[i], &cs[i]);
    const double sphi = 2.0 * sn[i] * cs[i], omc = 2.0 * sn[i] * sn[i];
    const V3 dh = F.dh[i];
    const V3 xd = cross(om, dh), xdd = cross(xd, dh);
    const V3 si = v3(om.x + sphi * xd.x + omc * xdd.x, om.y + sphi * xd.y + omc * xdd.y, om.z + sphi * xd.z + omc * xdd.z);   // rotation by -phi about dh
    pk[(3 * (i + 1) + 0) * ldp] = si.x; pk[(3 * (i + 1) + 1) * ldp] = si.y; pk[(3 * (i + 1) + 2) * ldp] = si.z;
    om = fma3(dlam[i] * K.inv_so3_dt, F.d[i], si);
  }
  V3 bgyr = v3(0, 0, 0);
#pragma unroll
  for (int k = 0; k < 3; ++k) bgyr = fma3(cbg[k], W.bg[k], bgyr);
  const V3 g_raw = g_meas - bgyr;
  rg[0] = K.w_gyr * (om.x - (K.Mg[0] * g_raw.x + K.Mg[1] * g_raw.y + K.Mg[2] * g_raw.z));
  rg[1] = K.w_gyr * (om.y - (K.Mg[3] * g_raw.x + K.Mg[4] * g_raw.y + K.Mg[5] * g_raw.z));
  rg[2] = K.w_gyr * (om.z - (K.Mg[6] * g_raw.x + K.Mg[7] * g_raw.y + K.Mg[8] * g_raw.z));
  row0[GYR_RES_COL * ld] = rg[0];
#pragma unroll
  for (int c = GYR_RES_COL + 1; c < 24; ++c) row0[c * ld] = 0.0;
  pk[36 * ldp] = rg[1]; pk[37 * ldp] = rg[2];
  // d omega_k / d eps_j = y_j Jr^-1_j - Jr^-1_{j+1} y_{j+1},  y_i = lambda_i ((w_i x s_i) Jr(phi_i)) + lambda'_i w_i / dt   (w scaled by w_gyr)
  V3 w[3], zn[3];
  w[0] = v3(K.w_gyr, 0, 0); w[1] = v3(0, K.w_gyr, 0); w[2] = v3(0, 0, K.w_gyr);
#pragma unroll
  for (int r = 0; r < 3; ++r) zn[r] = v3(0, 0, 0);
#pragma unroll
  for (int i = 4; i >= 0; --i) {
    const double sphi = 2.0 * sn[i] * cs[i], omc = 2.0 * sn[i] * sn[i];
    const double c1 = omc * F.ith[i], c2 = lam[i] - sphi * F.ith[i], dl = dlam[i] * K.inv_so3_dt;
    const V3 dh = F.dh[i];
    const volatile double* sv = pk + 3 * (i + 1) * ldp;
    const V3 si = v3(sv[0], sv[ldp], sv[2 * ldp]);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const V3 x = cross(w[r], si);
      const V3 xd = cross(x, dh), xdd = cross(xd, dh);
      const V3 yv = v3(lam[i] * x.x - c1 * xd.x + c2 * xdd.x + dl * w[r].x, lam[i] * x.y - c1 * xd.y + c2 * xdd.y + dl * w[r].y, lam[i] * x.z - c1 * xd.z + c2 * xdd.z + dl * w[r].z);
      const V3 up = mulT(F.jri[i], yv) - zn[r];
      zn[r] = mul(F.jri[i], yv);
      const V3 wd = cross(w[r], dh), wdd = cross(wd, dh);
      w[r] = v3(w[r].x - sphi * wd.x + omc * wdd.x, w[r].y - sphi * wd.y + omc * wdd.y, w[r].z - sphi * wd.z + omc * wdd.z);   // exp(lambda d) w
      if (r == 0) { row0[(3 * (i + 1) + 0) * ld] = up.x; row0[(3 * (i + 1) + 1) * ld] = up.y; row0[(3 * (i + 1) + 2) * ld] = up.z; }
      else { pk[(18 * (r - 1) + 3 * (i + 1) + 0) * ldp] = up.x; pk[(18 * (r - 1) + 3 * (i + 1) + 1) * ldp] = up.y; pk[(18 * (r - 1) + 3 * (i + 1) + 2) * ldp] = up.z; }
    }
  }
  row0[0] = -zn[0].x; row0[ld] = -zn[0].y; row0[2 * ld] = -zn[0].z;
  pk[0] = -zn[1].x; pk[ldp] = -zn[1].y; pk[2 * ldp] = -zn[1].z;
  pk[18 * ldp] = -zn[2].x; pk[19 * ldp] = -zn[2].y; pk[20 * ldp] = -zn[2].z;
}
// park: rows 1 and 2 in the parked layout (the CPU test and the host harness)
ICC_HD void imu_gyro_rows(const ImuWin& W, const ImuConst& K, double u_so3, double u_bg, V3 g_meas, double* __restrict__ row0, int ld, double (&park)[GYR_PARK], double (&rg)[3]) {
  imu_gyro_rows(W, K, u_so3, u_bg, g_meas, row0, ld, park, 1, rg);
}

ICC_HD void imu_gyro_row_expand(const double (&park)[GYR_PARK], int k, double* __restrict__ row, int ld) {
#pragma unroll
  for (int c = 0; c < 18; ++c) row[c * ld] = k == 1 ? park[c] : park[18 + c];
  row[GYR_RES_COL * ld] = k == 1 ? park[36] : park[37];
#pragma unroll
  for (int c = GYR_RES_COL + 1; c < 24; ++c) row[c * ld] = 0.0;
}

}  // namespace icc
