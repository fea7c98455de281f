// Spline knot initialisation on the device (SURVEY §8(f) row f2, first half).
//
// Reference: SplineTrajectoryEstimator::BatchInitSO3R3VisPoses (core/spline_trajectory_estimator.impl.h:278-339) with
// utils::InterpolateQuaternions / InterpolateVector3d (src/utils/utils.cc:214-261), one thread per knot: so3_knot / r3_knot
// (icc_rotinit_math.cuh), which a host-only handle runs on the CPU.  FindClosestTimestamp's linear scan becomes a bisection that picks
// the same index (nearest_sorted), Eigen's slerp is slerp4.  The kernel writes BOTH state copies of the handle (current / candidate) in
// their padded double4 layout, so no knot ever crosses PCIe.
#include "icc_kernels.h"
#include "icc_rotinit_math.cuh"

namespace icc {

namespace {

__global__ void init_knots_kernel(int nv, const double* __restrict__ t_vis, const double* __restrict__ q_wc, const double* __restrict__ p_wc, Q4 q_ci, V3 t_ci,
                                  int nso3, int64_t dt_so3_ns, int nr3, int64_t dt_r3_ns, double4* so3_a, double4* so3_b, double4* r3_a, double4* r3_b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nso3) {
    const double4 o = so3_knot(i, dt_so3_ns, nv, t_vis, q_wc, p_wc, q_ci, t_ci);
    so3_a[i] = o; so3_b[i] = o;
  } else if (i < nso3 + nr3) {
    const int j = i - nso3;
    const double4 o = r3_knot(j, dt_r3_ns, nr3, nv, t_vis, q_wc, p_wc, q_ci, t_ci);
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
