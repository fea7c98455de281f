// Small dense linear algebra that runs per thread: the one Cholesky of the pose / board-point, camera calibration and static IMU
// kernels, and the matrix-to-quaternion rule of the pose kernels.  Kept __host__ __device__ in a header so that
// tests/test_host_device_math.py can compile exactly this code for the CPU.
#pragma once
#include "icc_device_math.cuh"

namespace icc {

// In-place Cholesky factor (lower triangle) of the symmetric N x N matrix A, in registers.  A non-positive pivot is replaced by 1, the
// factorisation runs to the end (finite entries) and false is returned: the matrix was not positive definite.
template <int N>
ICC_HD bool chol_factor(double (&A)[N][N]) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double d = A[j][j];
#pragma unroll
    for (int k = 0; k < N; ++k) if (k < j) d -= A[j][k] * A[j][k];
    if (!(d > 0.0)) { ok = false; d = 1.0; }
    const double l = sqrt(d), il = 1.0 / l;
    A[j][j] = l;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if (i > j) {
        double s = A[i][j];
#pragma unroll
        for (int k = 0; k < N; ++k) if (k < j) s -= A[i][k] * A[j][k];
        A[i][j] = s * il;
      }
    }
  }
  return ok;
}

// b <- A^-1 b by forward and backward substitution with the factor chol_factor left in A
template <int N>
ICC_HD void chol_substitute(const double (&A)[N][N], double (&b)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < N; ++k) if (k < i) s -= A[i][k] * b[k];
    b[i] = s / A[i][i];
  }
#pragma unroll
  for (int ii = 0; ii < N; ++ii) {
    const int i = N - 1 - ii;
    double s = b[i];
#pragma unroll
    for (int k = 0; k < N; ++k) if (k > i) s -= A[k][i] * b[k];
    b[i] = s / A[i][i];
  }
}

// Cholesky solve of the symmetric positive definite N x N system (A lower triangle used); false if not SPD
template <int N>
ICC_HD bool chol_solve(double (&A)[N][N], double (&b)[N]) {
  const bool ok = chol_factor<N>(A);
  chol_substitute<N>(A, b);
  return ok;
}

ICC_HD Q4 quat_from_columns(V3 r1, V3 r2, V3 r3) {   // rotation matrix with columns r1 r2 r3 -> unit quaternion
  const double m00 = r1.x, m10 = r1.y, m20 = r1.z, m01 = r2.x, m11 = r2.y, m21 = r2.z, m02 = r3.x, m12 = r3.y, m22 = r3.z;
  const double tr = m00 + m11 + m22;
  Q4 q;
  if (tr > 0.0) { const double s = sqrt(tr + 1.0) * 2.0; q = q4((m21 - m12) / s, (m02 - m20) / s, (m10 - m01) / s, 0.25 * s); }
  else if (m00 > m11 && m00 > m22) { const double s = sqrt(1.0 + m00 - m11 - m22) * 2.0; q = q4(0.25 * s, (m01 + m10) / s, (m02 + m20) / s, (m21 - m12) / s); }
  else if (m11 > m22) { const double s = sqrt(1.0 + m11 - m00 - m22) * 2.0; q = q4((m01 + m10) / s, 0.25 * s, (m12 + m21) / s, (m02 - m20) / s); }
  else { const double s = sqrt(1.0 + m22 - m00 - m11) * 2.0; q = q4((m02 + m20) / s, (m12 + m21) / s, 0.25 * s, (m10 - m01) / s); }
  return qnormalized(q);
}

}  // namespace icc
