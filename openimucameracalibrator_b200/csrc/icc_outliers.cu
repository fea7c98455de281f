// Outlier corners between spline solves (icc_get_corner_errors / icc_reject_outlier_corners, icc_api.cu).
//
// The residual pairs come from the cost-only vision kernel (icc_eval.cu) at the current state, so a corner's error is exactly the pair
// icc_evaluate reports for it.  Three passes follow on the device:
//   corner_error_kernel  e = sqrt(rx^2 + ry^2) per corner; sum e^2, count and failed projections, one warp sum and one atomic per warp
//   keep_count_kernel    one warp per frame: ballot + popc of the keep mask
//   scan_counts_kernel   one CTA: exclusive scan of the kept counts into the new frame offsets
//   compact_kernel       one warp per frame: ballot prefix over the keep mask, kept corners written in order
// The rule (rx == 0 || ry == 0: not counted, kept -- impl.h:1058-1064; the 1e10 pair of a failed projection: not counted, rejected;
// otherwise rejected iff e > threshold) is corner_kept below, and icc_api.cu only ever sees the per-frame counts.
#include "icc_kernels.h"
#include "icc_reduce.cuh"

namespace icc {
namespace {

ICC_D bool pair_is_zero(double r0, double r1) { return r0 == 0.0 || r1 == 0.0; }
ICC_D bool pair_failed(double r0, double r1) { return r0 == 1e10 && r1 == 1e10; }   // residuals.h:391-398 (and the tangent residual's b.p <= 0)

ICC_D bool corner_kept(double2 r, double e, double thr) {
  if (pair_is_zero(r.x, r.y)) return true;
  if (pair_failed(r.x, r.y)) return false;
  return !(e > thr);
}

__global__ void corner_error_kernel(int n, const double2* __restrict__ res, double* __restrict__ err, double* __restrict__ sums) {
  double s2 = 0.0, cnt = 0.0, failed = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += stride) {
    const double2 r = res[c];
    const double e = sqrt(r.x * r.x + r.y * r.y);
    err[c] = e;
    if (pair_is_zero(r.x, r.y)) continue;
    if (pair_failed(r.x, r.y)) { failed += 1.0; continue; }
    s2 += e * e; cnt += 1.0;
  }
  s2 = warp_sum(s2); cnt = warp_sum(cnt); failed = warp_sum(failed);
  if ((threadIdx.x & 31) == 0) { atomicAdd(sums, s2); atomicAdd(sums + 1, cnt); atomicAdd(sums + 2, failed); }
}

__global__ void keep_count_kernel(int n_frames, const int* __restrict__ f_off, const double2* __restrict__ res, const double* __restrict__ err, double thr,
                                  int* __restrict__ kept) {
  const int lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  for (int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); f < n_frames; f += warps) {
    int k = 0;
    for (int base = f_off[f]; base < f_off[f + 1]; base += 32) {
      const int c = base + lane;
      const bool keep = c < f_off[f + 1] && corner_kept(res[c], err[c], thr);
      k += __popc(__ballot_sync(0xffffffffu, keep));
    }
    if (lane == 0) kept[f] = k;
  }
}

// off[0] = 0, off[f + 1] = off[f] + kept[f]; one CTA of 1024 threads walks the frames in tiles of 1024
__global__ void __launch_bounds__(1024) scan_counts_kernel(int n_frames, const int* __restrict__ kept, int* __restrict__ off) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { carry = 0; off[0] = 0; }
  __syncthreads();
  for (int base = 0; base < n_frames; base += 1024) {
    const int f = base + threadIdx.x;
    const int v = f < n_frames ? kept[f] : 0;
    int x = v;   // inclusive scan in the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int t = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
      warp_tot[lane] = t;   // inclusive over the warps
    }
    __syncthreads();
    const int incl = carry + (warp ? warp_tot[warp - 1] : 0) + x;
    if (f < n_frames) off[f + 1] = incl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
}

// src_in == nullptr: the corners still lie as assembled, frame f's first one being input corner in_off[f]
__global__ void compact_kernel(int n_frames, const int* __restrict__ off_old, const int* __restrict__ off_new, const double2* __restrict__ res,
                               const double* __restrict__ err, double thr, const double2* __restrict__ uv_in, const int* __restrict__ pid_in,
                               const double4* __restrict__ bear_in, const int* __restrict__ bear_ok_in, const int* __restrict__ src_in,
                               const int* __restrict__ in_off, double2* __restrict__ uv_out, int* __restrict__ pid_out, double4* __restrict__ bear_out,
                               int* __restrict__ bear_ok_out, int* __restrict__ src_out) {
  const int lane = threadIdx.x & 31, warps = gridDim.x * (blockDim.x >> 5);
  const unsigned below = (1u << lane) - 1u;
  for (int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); f < n_frames; f += warps) {
    const int c0 = off_old[f], c1 = off_old[f + 1];
    int dst = off_new[f];
    for (int base = c0; base < c1; base += 32) {
      const int c = base + lane;
      const bool keep = c < c1 && corner_kept(res[c], err[c], thr);
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int o = dst + __popc(m & below);
        uv_out[o] = uv_in[c]; pid_out[o] = pid_in[c];
        if (bear_out) { bear_out[o] = bear_in[c]; bear_ok_out[o] = bear_ok_in[c]; }
        src_out[o] = src_in ? src_in[c] : in_off[f] + (c - c0);
      }
      dst += __popc(m);
    }
  }
}

int warp_grid(int n_units) { const int b = (n_units + 7) / 8; return b < 1 ? 1 : (b > 4096 ? 4096 : b); }   // 8 warps per CTA

}  // namespace

void launch_corner_errors(int n, const double* res2, double* err, double* sums, cudaStream_t st) {
  if (n <= 0) return;
  const int blocks = (n + 255) / 256;
  corner_error_kernel<<<blocks < 2048 ? blocks : 2048, 256, 0, st>>>(n, reinterpret_cast<const double2*>(res2), err, sums);
  count_launch();
}

void launch_compact_corners(const CornerCompaction& C, cudaStream_t st) {
  if (C.n_frames <= 0) return;
  const double2* res = reinterpret_cast<const double2*>(C.res2);
  keep_count_kernel<<<warp_grid(C.n_frames), 256, 0, st>>>(C.n_frames, C.off_old, res, C.err, C.threshold, C.kept);
  count_launch();
  scan_counts_kernel<<<1, 1024, 0, st>>>(C.n_frames, C.kept, C.off_new);
  count_launch();
  compact_kernel<<<warp_grid(C.n_frames), 256, 0, st>>>(C.n_frames, C.off_old, C.off_new, res, C.err, C.threshold, C.uv_in, C.pid_in, C.bear_in, C.bear_ok_in,
                                                       C.src_in, C.in_off, C.uv_out, C.pid_out, C.bear_out, C.bear_ok_out, C.src_out);
  count_launch();
}

}  // namespace icc
