// ORACLE — TEST INFRASTRUCTURE ONLY.  Never linked into, imported by, or called from the
// product path (openimucameracalibrator_b200/).  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may use it.
//
// CPU restatement (FP64, dependency free) of the scalar-templated math that the reference's
// continuous-time IMU-camera calibration evaluates through Ceres Jets:
//   * forward-mode dual number            ~ ceres::Jet<double,4>  (ceres-solver 2.1.0, external)
//   * SO(3)/SE(3) on unit quaternions     ~ third_party/Sophus/sophus/so3.hpp:247-290,326-339,359-370,584-620
//                                           third_party/Sophus/sophus/se3.hpp:135-200,761-783
//   * uniform B-spline blending matrices  ~ include/OpenCameraCalibrator/basalt_spline/spline_common.h:67-133
//   * cumulative SO(3) / R^3 spline eval  ~ include/OpenCameraCalibrator/basalt_spline/ceres_spline_helper.h:69-220
//   * IMU triad model                     ~ include/OpenCameraCalibrator/utils/types.h:226-246,304-307
//   * camera projections                  ~ TheiaSfM camera models (pyTheiaSfM@69c3d37, NOT in the reference's repository):
//                                           restated from the published model equations; call sites
//                                           basalt_spline/ceres_calib_split_residuals.h:247-270,366-389
//
// PARITY UNPINNED: the reference ships no tests / golden vectors for this path and cannot be built
// offline (Ceres, Theia, Eigen absent).  The restatement is pinned instead by (i) the known-answer
// blending matrices listed in SURVEY.md §8(a2), (ii) central finite differences of its own duals,
// (iii) an independent numpy implementation in the synthetic-data generator (tests/).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace icco {

// ----------------------------------------------------------------------------------------------
// Forward-mode dual number with W derivative lanes (Ceres evaluates DynamicAutoDiff in strides of 4).
// ----------------------------------------------------------------------------------------------
template <int W>
struct Jet {
  double a;
  double v[W];
  Jet() : a(0) { for (int i = 0; i < W; ++i) v[i] = 0; }
  Jet(double s) : a(s) { for (int i = 0; i < W; ++i) v[i] = 0; }  // NOLINT implicit by design
};
template <int W> inline Jet<W> operator+(const Jet<W>& x, const Jet<W>& y) { Jet<W> r; r.a = x.a + y.a; for (int i = 0; i < W; ++i) r.v[i] = x.v[i] + y.v[i]; return r; }
template <int W> inline Jet<W> operator-(const Jet<W>& x, const Jet<W>& y) { Jet<W> r; r.a = x.a - y.a; for (int i = 0; i < W; ++i) r.v[i] = x.v[i] - y.v[i]; return r; }
template <int W> inline Jet<W> operator-(const Jet<W>& x) { Jet<W> r; r.a = -x.a; for (int i = 0; i < W; ++i) r.v[i] = -x.v[i]; return r; }
template <int W> inline Jet<W> operator*(const Jet<W>& x, const Jet<W>& y) { Jet<W> r; r.a = x.a * y.a; for (int i = 0; i < W; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a; return r; }
template <int W> inline Jet<W> operator/(const Jet<W>& x, const Jet<W>& y) { Jet<W> r; const double inv = 1.0 / y.a; r.a = x.a * inv; for (int i = 0; i < W; ++i) r.v[i] = (x.v[i] - r.a * y.v[i]) * inv; return r; }
template <int W> inline Jet<W> operator+(const Jet<W>& x, double s) { Jet<W> r = x; r.a += s; return r; }
template <int W> inline Jet<W> operator+(double s, const Jet<W>& x) { return x + s; }
template <int W> inline Jet<W> operator-(const Jet<W>& x, double s) { Jet<W> r = x; r.a -= s; return r; }
template <int W> inline Jet<W> operator-(double s, const Jet<W>& x) { return -x + s; }
template <int W> inline Jet<W> operator*(const Jet<W>& x, double s) { Jet<W> r; r.a = x.a * s; for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * s; return r; }
template <int W> inline Jet<W> operator*(double s, const Jet<W>& x) { return x * s; }
template <int W> inline Jet<W> operator/(const Jet<W>& x, double s) { return x * (1.0 / s); }
template <int W> inline Jet<W> operator/(double s, const Jet<W>& y) { return Jet<W>(s) / y; }
template <int W> inline Jet<W>& operator+=(Jet<W>& x, const Jet<W>& y) { x = x + y; return x; }
template <int W> inline Jet<W>& operator-=(Jet<W>& x, const Jet<W>& y) { x = x - y; return x; }
template <int W> inline Jet<W>& operator*=(Jet<W>& x, const Jet<W>& y) { x = x * y; return x; }
template <int W> inline bool operator<(const Jet<W>& x, const Jet<W>& y) { return x.a < y.a; }
template <int W> inline bool operator>(const Jet<W>& x, const Jet<W>& y) { return x.a > y.a; }
template <int W> inline bool operator<=(const Jet<W>& x, const Jet<W>& y) { return x.a <= y.a; }
template <int W> inline bool operator>=(const Jet<W>& x, const Jet<W>& y) { return x.a >= y.a; }
template <int W> inline bool operator<(const Jet<W>& x, double y) { return x.a < y; }
template <int W> inline bool operator>(const Jet<W>& x, double y) { return x.a > y; }
template <int W> inline bool operator<=(const Jet<W>& x, double y) { return x.a <= y; }
template <int W> inline bool operator>=(const Jet<W>& x, double y) { return x.a >= y; }

inline double jsqrt(double x) { return std::sqrt(x); }
inline double jsin(double x) { return std::sin(x); }
inline double jcos(double x) { return std::cos(x); }
inline double jatan(double x) { return std::atan(x); }
inline double jatan2(double y, double x) { return std::atan2(y, x); }
inline double jabs(double x) { return std::fabs(x); }
inline double jtan(double x) { return std::tan(x); }
inline double jval(double x) { return x; }
template <int W> inline Jet<W> jsqrt(const Jet<W>& x) { Jet<W> r; r.a = std::sqrt(x.a); const double d = 0.5 / r.a; for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * d; return r; }
template <int W> inline Jet<W> jsin(const Jet<W>& x) { Jet<W> r; r.a = std::sin(x.a); const double d = std::cos(x.a); for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * d; return r; }
template <int W> inline Jet<W> jcos(const Jet<W>& x) { Jet<W> r; r.a = std::cos(x.a); const double d = -std::sin(x.a); for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * d; return r; }
template <int W> inline Jet<W> jtan(const Jet<W>& x) { Jet<W> r; r.a = std::tan(x.a); const double d = 1.0 + r.a * r.a; for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * d; return r; }
template <int W> inline Jet<W> jatan(const Jet<W>& x) { Jet<W> r; r.a = std::atan(x.a); const double d = 1.0 / (1.0 + x.a * x.a); for (int i = 0; i < W; ++i) r.v[i] = x.v[i] * d; return r; }
template <int W> inline Jet<W> jatan2(const Jet<W>& y, const Jet<W>& x) { Jet<W> r; r.a = std::atan2(y.a, x.a); const double d = 1.0 / (x.a * x.a + y.a * y.a); for (int i = 0; i < W; ++i) r.v[i] = (x.a * y.v[i] - y.a * x.v[i]) * d; return r; }
template <int W> inline Jet<W> jabs(const Jet<W>& x) { return x.a < 0.0 ? -x : x; }
template <int W> inline double jval(const Jet<W>& x) { return x.a; }

// ----------------------------------------------------------------------------------------------
// Small fixed-size algebra.
// ----------------------------------------------------------------------------------------------
template <class T> struct V3 { T x, y, z; };
template <class T> struct Q4 { T x, y, z, w; };          // storage order x,y,z,w  (so3.hpp:218-225)
template <class T> struct M3 { T m[3][3]; };

template <class T> inline V3<T> operator+(const V3<T>& a, const V3<T>& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class T> inline V3<T> operator-(const V3<T>& a, const V3<T>& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> inline V3<T> operator*(const V3<T>& a, const T& s) { return {a.x * s, a.y * s, a.z * s}; }
template <class T> inline V3<T> cross(const V3<T>& a, const V3<T>& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
template <class T> inline T dot(const V3<T>& a, const V3<T>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <class T> inline V3<T> mul(const M3<T>& A, const V3<T>& b) {
  return {A.m[0][0] * b.x + A.m[0][1] * b.y + A.m[0][2] * b.z,
          A.m[1][0] * b.x + A.m[1][1] * b.y + A.m[1][2] * b.z,
          A.m[2][0] * b.x + A.m[2][1] * b.y + A.m[2][2] * b.z};
}

constexpr double kSophusEps = 1e-10;  // third_party/Sophus/sophus/common.hpp:94

// SO3(quaternion) constructor re-normalises (so3.hpp:480-487); product and inverse go through it.
template <class T> inline Q4<T> qnormalized(const Q4<T>& q) {
  T n = jsqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
// so3.hpp:326-339 (explicit Hamilton product, then SO3(quat) -> normalize)
template <class T> inline Q4<T> so3_mul(const Q4<T>& a, const Q4<T>& b) {
  Q4<T> r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return qnormalized(r);
}
// so3.hpp:225-227 inverse = SO3(conjugate) -> normalize
template <class T> inline Q4<T> so3_inv(const Q4<T>& a) { return qnormalized(Q4<T>{-a.x, -a.y, -a.z, a.w}); }
// so3.hpp:359-370 point action  p + w*uv + qv x uv, uv = 2 (qv x p)
template <class T> inline V3<T> so3_act(const Q4<T>& q, const V3<T>& p) {
  V3<T> qv{q.x, q.y, q.z};
  V3<T> uv = cross(qv, p);
  uv = uv + uv;
  return p + uv * q.w + cross(qv, uv);
}
// Eigen::QuaternionBase::toRotationMatrix (used by SO3::matrix()/Adj() and SE3::matrix()).
template <class T> inline M3<T> so3_matrix(const Q4<T>& q) {
  const T tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
  const T twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const T txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const T tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  M3<T> R;
  R.m[0][0] = 1.0 - (tyy + tzz); R.m[0][1] = txy - twz;         R.m[0][2] = txz + twy;
  R.m[1][0] = txy + twz;         R.m[1][1] = 1.0 - (txx + tzz); R.m[1][2] = tyz - twx;
  R.m[2][0] = txz - twy;         R.m[2][1] = tyz + twx;         R.m[2][2] = 1.0 - (txx + tyy);
  return R;
}
// so3.hpp:584-620 expAndTheta
template <class T> inline Q4<T> so3_exp(const V3<T>& omega, T* theta_out = nullptr) {
  const T theta_sq = dot(omega, omega);
  T imag_factor, real_factor, theta;
  if (theta_sq < kSophusEps * kSophusEps) {
    theta = T(0.0);
    const T theta_po4 = theta_sq * theta_sq;
    imag_factor = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * theta_po4;
    real_factor = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * theta_po4;
  } else {
    theta = jsqrt(theta_sq);
    const T half_theta = 0.5 * theta;
    imag_factor = jsin(half_theta) / theta;
    real_factor = jcos(half_theta);
  }
  if (theta_out) *theta_out = theta;
  return {imag_factor * omega.x, imag_factor * omega.y, imag_factor * omega.z, real_factor};
}
// so3.hpp:247-290 logAndTheta (atan based)
template <class T> inline V3<T> so3_log(const Q4<T>& q) {
  const T squared_n = q.x * q.x + q.y * q.y + q.z * q.z;
  const T w = q.w;
  T two_atan_nbyw_by_n;
  if (squared_n < kSophusEps * kSophusEps) {
    const T squared_w = w * w;
    two_atan_nbyw_by_n = 2.0 / w - (2.0 / 3.0) * squared_n / (w * squared_w);
  } else {
    const T n = jsqrt(squared_n);
    if (jabs(w) < kSophusEps) {
      if (w > 0.0) two_atan_nbyw_by_n = M_PI / n; else two_atan_nbyw_by_n = -M_PI / n;
    } else {
      two_atan_nbyw_by_n = 2.0 * jatan(n / w) / n;
    }
  }
  return {two_atan_nbyw_by_n * q.x, two_atan_nbyw_by_n * q.y, two_atan_nbyw_by_n * q.z};
}

// SE3 stored as quaternion(4) then translation(3) (spline_trajectory_estimator.impl.h:519,579).
template <class T> struct SE3T { Q4<T> q; V3<T> t; };
template <class T> inline SE3T<T> se3_mul(const SE3T<T>& a, const SE3T<T>& b) { return {so3_mul(a.q, b.q), a.t + so3_act(a.q, b.t)}; }
template <class T> inline SE3T<T> se3_inv(const SE3T<T>& a) { Q4<T> qi = so3_inv(a.q); V3<T> nt{-a.t.x, -a.t.y, -a.t.z}; return {qi, so3_act(qi, nt)}; }
// se3.hpp:761-783 coupled exponential, tangent = (upsilon, omega)
inline SE3T<double> se3_exp(const double a[6]) {
  V3<double> ups{a[0], a[1], a[2]}, om{a[3], a[4], a[5]};
  double theta;
  Q4<double> q = so3_exp(om, &theta);
  M3<double> V;
  if (theta < kSophusEps) {
    V = so3_matrix(q);
  } else {
    const double th2 = theta * theta;
    const double A = (1.0 - std::cos(theta)) / th2, B = (theta - std::sin(theta)) / (th2 * theta);
    const double O[3][3] = {{0, -om.z, om.y}, {om.z, 0, -om.x}, {-om.y, om.x, 0}};
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
      double o2 = 0; for (int k = 0; k < 3; ++k) o2 += O[i][k] * O[k][j];
      V.m[i][j] = (i == j ? 1.0 : 0.0) + A * O[i][j] + B * o2;
    }
  }
  return {q, mul(V, ups)};
}

// ----------------------------------------------------------------------------------------------
// Blending matrices (spline_common.h:67-133).  Row = knot index, column = power of u.
// ----------------------------------------------------------------------------------------------
inline uint64_t binom(uint64_t n, uint64_t k) { if (k > n) return 0; uint64_t r = 1; for (uint64_t d = 1; d <= k; ++d) { r *= n--; r /= d; } return r; }
template <int N> struct Blend {
  double M[N][N];    // non-cumulative
  double Mc[N][N];   // cumulative
  double base[N][N]; // derivative coefficients of the monomial vector
  Blend() {
    double m[N][N];
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) {
      double sum = 0;
      for (int s = j; s < N; ++s) sum += std::pow(-1.0, s - j) * double(binom(N, s - j)) * std::pow(N - s - 1.0, N - 1.0 - i);
      m[j][i] = double(binom(N - 1, N - 1 - i)) * sum;
    }
    uint64_t fact = 1; for (int i = 2; i < N; ++i) fact *= i;
    double mc[N][N];
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) mc[i][j] = m[i][j];
    for (int i = 0; i < N; ++i) for (int j = i + 1; j < N; ++j) for (int c = 0; c < N; ++c) mc[i][c] += m[j][c];
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) { M[i][j] = m[i][j] / double(fact); Mc[i][j] = mc[i][j] / double(fact); }
    for (int i = 0; i < N; ++i) for (int j = 0; j < N; ++j) base[i][j] = 0;
    for (int j = 0; j < N; ++j) base[0][j] = 1;
    const int DEG = N - 1; int order = DEG;
    for (int n = 1; n < N; ++n) { for (int i = DEG - order; i < N; ++i) base[n][i] = (order - DEG + i) * base[n - 1][i]; order--; }
  }
};
template <int N> inline const Blend<N>& blend() { static const Blend<N> b; return b; }

// ceres_spline_helper.h:69-87
template <int N, int D, class T> inline void base_coeffs_with_time(T res[N], const T& t) {
  const Blend<N>& B = blend<N>();
  for (int j = 0; j < N; ++j) res[j] = T(0.0);
  if (D < N) {
    res[D] = T(B.base[D][D]);
    T _t = t;
    for (int j = D + 1; j < N; ++j) { res[j] = B.base[D][j] * _t; _t = _t * t; }
  }
}
template <int N, class T> inline void matvec(const double M[N][N], const T p[N], T out[N]) {
  for (int i = 0; i < N; ++i) { T s(0.0); for (int j = 0; j < N; ++j) s = s + M[i][j] * p[j]; out[i] = s; }
}

// ceres_spline_helper.h:101-187 (value and body velocity; accel/jerk are unused by the live residuals)
template <int N, class T>
inline void evaluate_lie_so3(const T* const* knots, const T& u, const T& inv_dt, Q4<T>* rot_out, V3<T>* vel_out) {
  const Blend<N>& B = blend<N>();
  T p[N], coeff[N], dcoeff[N];
  base_coeffs_with_time<N, 0>(p, u);
  matvec<N>(B.Mc, p, coeff);
  if (vel_out) {
    base_coeffs_with_time<N, 1>(p, u);
    matvec<N>(B.Mc, p, dcoeff);
    for (int i = 0; i < N; ++i) dcoeff[i] = inv_dt * dcoeff[i];
  }
  Q4<T> res;
  if (rot_out) res = Q4<T>{knots[0][0], knots[0][1], knots[0][2], knots[0][3]};
  V3<T> rot_vel{T(0.0), T(0.0), T(0.0)};
  for (int i = 0; i < N - 1; ++i) {
    Q4<T> p0{knots[i][0], knots[i][1], knots[i][2], knots[i][3]};
    Q4<T> p1{knots[i + 1][0], knots[i + 1][1], knots[i + 1][2], knots[i + 1][3]};
    Q4<T> r01 = so3_mul(so3_inv(p0), p1);
    V3<T> delta = so3_log(r01);
    Q4<T> exp_kdelta = so3_exp(delta * coeff[i + 1]);
    if (rot_out) res = so3_mul(res, exp_kdelta);
    if (vel_out) {
      M3<T> A = so3_matrix(so3_inv(exp_kdelta));
      rot_vel = mul(A, rot_vel);
      rot_vel = rot_vel + delta * dcoeff[i + 1];
    }
  }
  if (rot_out) *rot_out = res;
  if (vel_out) *vel_out = rot_vel;
}

// ceres_spline_helper.h:198-220
template <int N, int DERIV, class T>
inline V3<T> evaluate_r3(const T* const* knots, const T& u, const T& inv_dt) {
  const Blend<N>& B = blend<N>();
  T p[N], coeff[N];
  base_coeffs_with_time<N, DERIV>(p, u);
  matvec<N>(B.M, p, coeff);
  T scale(1.0);
  for (int d = 0; d < DERIV; ++d) scale = scale * inv_dt;
  V3<T> out{T(0.0), T(0.0), T(0.0)};
  for (int i = 0; i < N; ++i) {
    const T c = scale * coeff[i];
    out.x = out.x + c * knots[i][0]; out.y = out.y + c * knots[i][1]; out.z = out.z + c * knots[i][2];
  }
  return out;
}

// utils/types.h:226-246,304-307: out = (mis * diag(s)) * (raw - bias)
template <class T>
inline V3<T> triad_unbias_normalize(const T& mis_yz, const T& mis_zy, const T& mis_zx, const T& mis_xz, const T& mis_xy,
                                    const T& mis_yx, const T& sx, const T& sy, const T& sz, const V3<T>& bias, const V3<T>& raw) {
  M3<T> mis;
  mis.m[0][0] = T(1.0); mis.m[0][1] = -mis_yz;  mis.m[0][2] = mis_zy;
  mis.m[1][0] = mis_xz; mis.m[1][1] = T(1.0);   mis.m[1][2] = -mis_zx;
  mis.m[2][0] = -mis_xy; mis.m[2][1] = mis_yx;  mis.m[2][2] = T(1.0);
  const T s[3] = {sx, sy, sz};
  M3<T> ms;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) ms.m[i][j] = mis.m[i][j] * s[j];
  return mul(ms, raw - bias);
}

// ----------------------------------------------------------------------------------------------
// Camera models: bool CameraToPixelCoordinates(intr, point3, pixel)  (Theia API contract).
// Model ids follow theia::CameraIntrinsicsModelType.
// ----------------------------------------------------------------------------------------------
enum CameraModel { PINHOLE = 0, PINHOLE_RADIAL_TANGENTIAL = 1, FISHEYE = 2, FOV = 3, DIVISION_UNDISTORTION = 4, DOUBLE_SPHERE = 5, EXTENDED_UNIFIED = 6 };
inline int camera_num_params(int model) {
  switch (model) { case PINHOLE: return 7; case PINHOLE_RADIAL_TANGENTIAL: return 10; case FISHEYE: return 9; case FOV: return 5;
                   case DIVISION_UNDISTORTION: return 5; case DOUBLE_SPHERE: return 7; case EXTENDED_UNIFIED: return 7; default: return -1; }
}

template <class T> inline bool project_pinhole(const T* k, const T* p, T* px) {  // [f, ar, skew, cx, cy, k1, k2]
  const T x = p[0] / p[2], y = p[1] / p[2];
  const T r2 = x * x + y * y;
  const T d = 1.0 + r2 * (k[5] + k[6] * r2);
  const T dx = x * d, dy = y * d;
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}
template <class T> inline bool project_pinhole_radtan(const T* k, const T* p, T* px) {  // [f, ar, skew, cx, cy, k1,k2,k3, t1,t2]
  const T x = p[0] / p[2], y = p[1] / p[2];
  const T r2 = x * x + y * y;
  const T d = 1.0 + r2 * (k[5] + r2 * (k[6] + r2 * k[7]));
  const T dx = x * d + 2.0 * k[8] * x * y + k[9] * (r2 + 2.0 * x * x);
  const T dy = y * d + 2.0 * k[9] * x * y + k[8] * (r2 + 2.0 * y * y);
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}
template <class T> inline bool project_fisheye(const T* k, const T* p, T* px) {  // [f, ar, skew, cx, cy, k1..k4]
  const T r2 = p[0] * p[0] + p[1] * p[1];
  T dx, dy;
  if (r2 < 1e-8) {
    dx = p[0]; dy = p[1];
  } else {
    const T r = jsqrt(r2);
    const T theta = jatan2(r, jabs(p[2]));
    const T th2 = theta * theta;
    const T theta_d = theta * (1.0 + th2 * (k[5] + th2 * (k[6] + th2 * (k[7] + th2 * k[8]))));
    dx = theta_d * p[0] / r; dy = theta_d * p[1] / r;
    if (p[2] < 0.0) { dx = -dx; dy = -dy; }
  }
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}
template <class T> inline bool project_fov(const T* k, const T* p, T* px) {  // [f, ar, cx, cy, omega]  (extension; not dispatched by the reference)
  const T x = p[0] / p[2], y = p[1] / p[2];
  const T r2 = x * x + y * y;
  const T om = k[4];
  T scale;
  if (om * om < 1e-10) {
    scale = T(1.0);
  } else if (r2 < 1e-10) {
    scale = 2.0 * jtan(0.5 * om) / om;
  } else {
    const T r = jsqrt(r2);
    scale = jatan(2.0 * r * jtan(0.5 * om)) / (om * r);
  }
  px[0] = k[0] * scale * x + k[2];
  px[1] = k[0] * k[1] * scale * y + k[3];
  return true;
}
template <class T> inline bool project_division_undistortion(const T* k, const T* p, T* px) {  // [f, ar, cx, cy, k]
  const T x = k[0] * (p[0] / p[2]), y = k[0] * k[1] * (p[1] / p[2]);
  const T r2 = x * x + y * y;
  const T denom = 2.0 * k[4] * r2;
  const T inner = 1.0 - 4.0 * k[4] * r2;
  if (jabs(denom) < 1e-15 || inner < 0.0) {
    px[0] = x; px[1] = y;
  } else {
    const T s = (1.0 - jsqrt(inner)) / denom;
    px[0] = x * s; px[1] = y * s;
  }
  px[0] = px[0] + k[2]; px[1] = px[1] + k[3];
  return true;
}
template <class T> inline T unified_w(const T& alpha) { return alpha > 0.5 ? (1.0 - alpha) / alpha : alpha / (1.0 - alpha); }
template <class T> inline bool project_double_sphere(const T* k, const T* p, T* px) {  // [f, ar, skew, cx, cy, xi, alpha]
  const T xi = k[5], alpha = k[6];
  const T r2 = p[0] * p[0] + p[1] * p[1];
  const T d1 = jsqrt(r2 + p[2] * p[2]);
  const T w1 = unified_w(alpha);
  const T w2 = (w1 + xi) / jsqrt(2.0 * w1 * xi + xi * xi + 1.0);
  if (p[2] <= -w2 * d1) return false;
  const T kk = xi * d1 + p[2];
  const T d2 = jsqrt(r2 + kk * kk);
  const T norm = alpha * d2 + (1.0 - alpha) * kk;
  const T dx = p[0] / norm, dy = p[1] / norm;
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}
template <class T> inline bool project_extended_unified(const T* k, const T* p, T* px) {  // [f, ar, skew, cx, cy, alpha, beta]
  const T alpha = k[5], beta = k[6];
  const T r2 = p[0] * p[0] + p[1] * p[1];
  const T rho = jsqrt(beta * r2 + p[2] * p[2]);
  const T norm = alpha * rho + (1.0 - alpha) * p[2];
  const T w = unified_w(alpha);
  if (p[2] <= -w * rho) return false;
  const T dx = p[0] / norm, dy = p[1] / norm;
  px[0] = k[0] * dx + k[2] * dy + k[3];
  px[1] = k[0] * k[1] * dy + k[4];
  return true;
}
// Dispatch mirrors ceres_calib_split_residuals.h:366-389.  `dispatch_fov` = false reproduces the reference
// (FOV falls through to success=false -> 1e10 residual); true enables the north-star FOV extension.
template <class T> inline bool project(int model, const T* k, const T* p, T* px, bool dispatch_fov) {
  switch (model) {
    case DIVISION_UNDISTORTION: return project_division_undistortion(k, p, px);
    case DOUBLE_SPHERE: return project_double_sphere(k, p, px);
    case PINHOLE: return project_pinhole(k, p, px);
    case FISHEYE: return project_fisheye(k, p, px);
    case EXTENDED_UNIFIED: return project_extended_unified(k, p, px);
    case PINHOLE_RADIAL_TANGENTIAL: return project_pinhole_radtan(k, p, px);
    case FOV: return dispatch_fov ? project_fov(k, p, px) : false;
    default: return false;
  }
}

}  // namespace icco
