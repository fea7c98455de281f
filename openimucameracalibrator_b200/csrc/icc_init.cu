// Spline knot initialisation on the device (SURVEY §8(f) row f2, first half).
//
// Reference: SplineTrajectoryEstimator::BatchInitSO3R3VisPoses (core/spline_trajectory_estimator.impl.h:278-339) with
// utils::InterpolateQuaternions / InterpolateVector3d (src/utils/utils.cc:214-261): every knot takes the pose of the view
// nearest to its ZERO-BASED knot time i * dt (quirk q7: compared with the absolute view timestamps), slerp / lerp towards the
// next view by dist / (t[k+1] - t[k]) -- always "forwards", whichever side of the view the knot time lies on -- where the pose is
// T_w_i = T_w_c T_i_c^-1 of the per-view prior.  One thread per knot; FindClosestTimestamp's linear scan becomes a bisection that
// picks the same index (icc_rotinit_math.cuh: nearest_sorted), Eigen's slerp is slerp4.  The kernel writes BOTH state copies of
// the handle (current / candidate) in their padded double4 layout, so no knot ever crosses PCIe.
#include "icc_kernels.h"
#include "icc_rotinit_math.cuh"

namespace icc {

namespace {

struct PoseD { Q4 q; V3 t; };
ICC_D PoseD view_T_w_i(const double* __restrict__ q_wc, const double* __restrict__ p_wc, int k, Q4 q_ci, V3 t_ci) {
  const Q4 qw = qnormalized(q4(q_wc[4 * k], q_wc[4 * k + 1], q_wc[4 * k + 2], q_wc[4 * k + 3]));
  PoseD r;
  r.q = qnormalized(qmul(qw, q_ci));                                                  // Sophus SE3 product re-normalises
  r.t = v3(p_wc[3 * k], p_wc[3 * k + 1], p_wc[3 * k + 2]) + qrot(qw, t_ci);
  return r;
}

__global__ void init_knots_kernel(int nv, const double* __restrict__ t_vis, const double* __restrict__ q_wc, const double* __restrict__ p_wc, Q4 q_ci, V3 t_ci,
                                  int nso3, int64_t dt_so3_ns, int nr3, int64_t dt_r3_ns, double4* so3_a, double4* so3_b, double4* r3_a, double4* r3_b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nso3) {                               // InterpolateQuaternions (utils.cc:214-241)
    const double t = double((int64_t)i * dt_so3_ns) * 1e-9;   // i * dt_so3_ns_ * NS_TO_S (impl.h:318): integer product first -- knot times tie with view mid-points, the rounding decides the nearest view
    double dist = 0.0;
    const int k = nearest_sorted(t_vis, nv, t, dist);
    const PoseD a = view_T_w_i(q_wc, p_wc, k, q_ci, t_ci);
    double4 q = make_double4(a.q.x, a.q.y, a.q.z, a.q.w);
    if (k < nv - 1) {
      const PoseD b = view_T_w_i(q_wc, p_wc, k + 1, q_ci, t_ci);
      q = slerp4(q, make_double4(b.q.x, b.q.y, b.q.z, b.q.w), dist / (t_vis[k + 1] - t_vis[k]));
    }
    const Q4 r = qnormalized(q4(q.x, q.y, q.z, q.w));     // Sophus::SO3d(quaternion) normalises
    const double4 o = make_double4(r.x, r.y, r.z, r.w);
    so3_a[i] = o; so3_b[i] = o;
  } else if (i < nso3 + nr3) {                  // InterpolateVector3d (utils.cc:243-261) incl. its `nearest < t_new.size()` test; the
    const int j = i - nso3;                     // reference's read past the last view falls back to the nearest value
    const double t = double((int64_t)j * dt_r3_ns) * 1e-9;
    double dist = 0.0;
    const int k = nearest_sorted(t_vis, nv, t, dist);
    const PoseD a = view_T_w_i(q_wc, p_wc, k, q_ci, t_ci);
    V3 p = a.t;
    if (k < nr3 && k + 1 < nv) {
      const PoseD b = view_T_w_i(q_wc, p_wc, k + 1, q_ci, t_ci);
      const double f = dist / (t_vis[k + 1] - t_vis[k]);
      p = v3((1.0 - f) * a.t.x + f * b.t.x, (1.0 - f) * a.t.y + f * b.t.y, (1.0 - f) * a.t.z + f * b.t.z);
    }
    const double4 o = make_double4(p.x, p.y, p.z, 0.0);
    r3_a[j] = o; r3_b[j] = o;
  }
}

// CalcTimes' relative sample time of the IMU stream: st = int64((t + offset) * 1e9) - start, the host's expression bit for bit (one rounded add,
// one rounded multiply -- nothing to contract --, truncation)
__global__ void imu_times_kernel(int n, const double* __restrict__ t_raw, double offset_s, int64_t start_ns, int64_t* __restrict__ st) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) st[i] = (int64_t)__dmul_rn(__dadd_rn(t_raw[i], offset_s), 1e9) - start_ns;
}

// smallest / largest corner point id (range check of batch_init_spline): out[0] = min(0, ids...), out[1] = max(-1, ids...)
__global__ void id_range_kernel(int n, const int* __restrict__ ids, int* out) {
  int lo = 0, hi = -1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { const int v = ids[i]; lo = min(lo, v); hi = max(hi, v); }
  for (int o = 16; o > 0; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
  if ((threadIdx.x & 31) == 0) { atomicMin(out, lo); atomicMax(out + 1, hi); }
}

}  // namespace

void launch_id_range(int n, const int* ids, int* out2, cudaStream_t st) {   // out2 must hold {0, -1} before the launch
  if (n <= 0) return;
  int grid = (n + 1023) / 1024; if (grid > 296) grid = 296;
  id_range_kernel<<<grid, 256, 0, st>>>(n, ids, out2);
  count_launch();
}

void launch_imu_times(int n, const double* t_raw, double offset_s, int64_t start_ns, int64_t* st_out, cudaStream_t st) {
  if (n <= 0) return;
  imu_times_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, t_raw, offset_s, start_ns, st_out);
  count_launch();
}

void launch_init_knots(int nv, const double* t_vis, const double* q_wc, const double* p_wc, const double T_c_i[7], int nso3, int64_t dt_so3_ns, int nr3, int64_t dt_r3_ns,
                       double4* so3_a, double4* so3_b, double4* r3_a, double4* r3_b, cudaStream_t st) {
  const int n = nso3 + nr3;
  if (n <= 0 || nv <= 0) return;
  init_knots_kernel<<<(n + 127) / 128, 128, 0, st>>>(nv, t_vis, q_wc, p_wc, q4(T_c_i[0], T_c_i[1], T_c_i[2], T_c_i[3]), v3(T_c_i[4], T_c_i[5], T_c_i[6]), nso3, dt_so3_ns, nr3, dt_r3_ns, so3_a, so3_b, r3_a, r3_b);
  count_launch();
}

}  // namespace icc
