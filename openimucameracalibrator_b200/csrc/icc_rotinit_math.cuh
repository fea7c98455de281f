// Scalar pieces of the rotation / time-offset initialiser (icc_rotinit.cu) and of the spline knot initialiser (icc_init.cu) that run per
// thread: kept __host__ __device__ in a header so that tests/test_host_device_math.py can compile exactly this code for the CPU
// (nearest-sample rule of the reference, Eigen's slerp, the dominant eigenvector behind the closed-form rotation), and so that a host-only
// handle (icc_api.cu) initialises its knots with the expressions init_knots_kernel runs.
#pragma once
#include "icc_device_math.cuh"

namespace icc {

// FindClosestTimestamp (utils.cc:194-212) on sorted times: first strict minimum of |t - ts[i]|
ICC_HD int nearest_sorted(const double* __restrict__ ts, int n, double t, double& dist) {
  int lo = 0, hi = n;                    // first index with ts >= t
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (ts[mid] < t) lo = mid + 1; else hi = mid; }
  int idx;
  if (lo == 0) idx = 0;
  else if (lo == n) idx = n - 1;
  else idx = (fabs(t - ts[lo - 1]) <= fabs(t - ts[lo])) ? lo - 1 : lo;
  dist = fabs(t - ts[idx]);
  return idx;
}

ICC_HD double4 slerp4(double4 a, double4 b, double t) {            // Eigen::Quaternion::slerp (utils.cc:234)
  const double thresh = 1.0 - 2.220446049250313e-16;
  const double d = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w, ad = fabs(d);
  double s0, s1;
  if (ad >= thresh) { s0 = 1.0 - t; s1 = t; }
  else { const double th = acos(ad), sth = sin(th); s0 = sin((1.0 - t) * th) / sth; s1 = sin(t * th) / sth; }
  if (d < 0) s1 = -s1;
  return make_double4(s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z, s0 * a.w + s1 * b.w);
}

// ---- BatchInitSO3R3VisPoses (impl.h:278-339), one knot per call -------------------------------------------------------------------------
// Every knot takes the pose of the view nearest to its ZERO-BASED knot time i * dt (quirk q7: compared with the absolute view timestamps)
// and slerps / lerps towards the next view by dist / (t[k+1] - t[k]) -- always "forwards", whichever side of the view the knot time lies
// on.  t_vis / q_wc / p_wc: the per-view priors in time order, T_c_i = (q_ci, t_ci).
struct Pose { Q4 q; V3 t; };

// T_w_i = T_w_c T_i_c^-1 of view k
ICC_HD Pose view_T_w_i(const double* __restrict__ q_wc, const double* __restrict__ p_wc, int k, Q4 q_ci, V3 t_ci) {
  const Q4 qw = qnormalized(q4(q_wc[4 * k], q_wc[4 * k + 1], q_wc[4 * k + 2], q_wc[4 * k + 3]));
  Pose r;
  r.q = qnormalized(qmul(qw, q_ci));                                                  // Sophus SE3 product re-normalises
  r.t = v3(p_wc[3 * k], p_wc[3 * k + 1], p_wc[3 * k + 2]) + qrot(qw, t_ci);
  return r;
}

// InterpolateQuaternions (utils.cc:214-241): SO(3) knot i as (x, y, z, w)
ICC_HD double4 so3_knot(int i, int64_t dt_ns, int nv, const double* __restrict__ t_vis, const double* __restrict__ q_wc, const double* __restrict__ p_wc,
                        Q4 q_ci, V3 t_ci) {
  const double t = double((int64_t)i * dt_ns) * 1e-9;   // i * dt_so3_ns_ * NS_TO_S (impl.h:318): integer product first -- knot times tie with view mid-points, the rounding decides the nearest view
  double dist = 0.0;
  const int k = nearest_sorted(t_vis, nv, t, dist);
  const Pose a = view_T_w_i(q_wc, p_wc, k, q_ci, t_ci);
  double4 q = make_double4(a.q.x, a.q.y, a.q.z, a.q.w);
  if (k < nv - 1) {
    const Pose b = view_T_w_i(q_wc, p_wc, k + 1, q_ci, t_ci);
    q = slerp4(q, make_double4(b.q.x, b.q.y, b.q.z, b.q.w), dist / (t_vis[k + 1] - t_vis[k]));
  }
  const Q4 r = qnormalized(q4(q.x, q.y, q.z, q.w));     // Sophus::SO3d(quaternion) normalises
  return make_double4(r.x, r.y, r.z, r.w);
}

// InterpolateVector3d (utils.cc:243-261): R³ knot j as (x, y, z, 0), incl. the reference's `nearest < t_new.size()` test (t_new: the
// nr3 knots); its read past the last view falls back to the nearest value
ICC_HD double4 r3_knot(int j, int64_t dt_ns, int nr3, int nv, const double* __restrict__ t_vis, const double* __restrict__ q_wc, const double* __restrict__ p_wc,
                       Q4 q_ci, V3 t_ci) {
  const double t = double((int64_t)j * dt_ns) * 1e-9;
  double dist = 0.0;
  const int k = nearest_sorted(t_vis, nv, t, dist);
  const Pose a = view_T_w_i(q_wc, p_wc, k, q_ci, t_ci);
  V3 p = a.t;
  if (k < nr3 && k + 1 < nv) {
    const Pose b = view_T_w_i(q_wc, p_wc, k + 1, q_ci, t_ci);
    const double f = dist / (t_vis[k + 1] - t_vis[k]);
    p = v3((1.0 - f) * a.t.x + f * b.t.x, (1.0 - f) * a.t.y + f * b.t.y, (1.0 - f) * a.t.z + f * b.t.z);
  }
  return make_double4(p.x, p.y, p.z, 0.0);
}

// largest eigenvector of the symmetric 4x4 matrix N by cyclic Jacobi rotations
ICC_HD void eig4_max(double (&A)[4][4], double (&qv)[4]) {
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 4; ++p) for (int q = p + 1; q < 4; ++q) off += A[p][q] * A[p][q];
    if (off < 1e-300) break;
    for (int p = 0; p < 4; ++p) for (int q = p + 1; q < 4; ++q) {
      if (fabs(A[p][q]) < 1e-300) continue;
      const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
      const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
      for (int k = 0; k < 4; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = cs * akp - sn * akq; A[k][q] = sn * akp + cs * akq; }
      for (int k = 0; k < 4; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = cs * apk - sn * aqk; A[q][k] = sn * apk + cs * aqk; }
      for (int k = 0; k < 4; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = cs * vkp - sn * vkq; V[k][q] = sn * vkp + cs * vkq; }
    }
  }
  int best = 0;
  for (int k = 1; k < 4; ++k) if (A[k][k] > A[best][best]) best = k;
  for (int k = 0; k < 4; ++k) qv[k] = V[k][best];
}

}  // namespace icc
