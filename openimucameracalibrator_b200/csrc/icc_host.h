// Host-side helpers shared by the drivers in the .cu files of libicc_b200.so, and the drivers the C-ABI shims of icc_api.cu call.
// Host code only: no device header includes this file.
#pragma once
#include "../../include/icc_b200.h"
#include "icc_kernels.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

// A failed CUDA call returns ICC_ERR_CUDA from the enclosing function and leaves "<call>: <CUDA error string>" in `sink`.
#define ICC_CUDA_CHECK(call, sink) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { (sink) = std::string(#call) + ": " + cudaGetErrorString(e__); return ICC_ERR_CUDA; } } while (0)

namespace icc {

// Process-wide caching allocator for device blocks: a calibration job allocates ~30 buffers and the CUDA driver's
// cudaMalloc / cudaFree cost 0.1-1 ms each, which would dominate the whole-job wall clock of back-to-back jobs.
// Freed blocks are kept (per device) and handed out again best-fit; icc_trim_device_cache() returns them to the driver.
struct BlockCache {
  std::mutex mu;
  std::multimap<size_t, std::pair<int, void*>> free_blocks;   // bytes -> (device, ptr)
  cudaError_t get(size_t bytes, void** out) {
    int dev = 0; cudaGetDevice(&dev);
    {
      std::lock_guard<std::mutex> lk(mu);
      for (auto it = free_blocks.lower_bound(bytes); it != free_blocks.end() && it->first <= 2 * bytes + 4096; ++it)
        if (it->second.first == dev) { *out = it->second.second; free_blocks.erase(it); return cudaSuccess; }
    }
    return cudaMalloc(out, bytes);
  }
  void put(size_t bytes, void* p) { int dev = 0; cudaGetDevice(&dev); std::lock_guard<std::mutex> lk(mu); free_blocks.emplace(bytes, std::make_pair(dev, p)); }
  void trim() { std::lock_guard<std::mutex> lk(mu); for (auto& kv : free_blocks) { cudaSetDevice(kv.second.first); cudaFree(kv.second.second); } free_blocks.clear(); }
};
inline BlockCache& block_cache() { static BlockCache* c = new BlockCache(); return *c; }   // intentionally leaked: outlives every handle

template <class T>
struct DevBuf {
  T* p = nullptr; size_t n = 0, cap_bytes = 0;
  ~DevBuf() { release(); }
  void release() { if (p) block_cache().put(cap_bytes, p); p = nullptr; n = 0; cap_bytes = 0; }
  cudaError_t alloc(size_t count) {
    const size_t bytes = (count * sizeof(T) + 255) / 256 * 256;
    if (p && cap_bytes >= bytes) { n = count; return cudaSuccess; }
    release(); n = count; if (!count) return cudaSuccess;
    void* q = nullptr; cudaError_t e = block_cache().get(bytes, &q); if (e != cudaSuccess) { n = 0; return e; }
    p = static_cast<T*>(q); cap_bytes = bytes; return cudaSuccess;
  }
  cudaError_t upload(const std::vector<T>& v) { cudaError_t e = alloc(v.size()); if (e != cudaSuccess || v.empty()) return e; return cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice); }
  // count elements from host memory, asynchronously on st
  cudaError_t upload(const void* src, size_t count, cudaStream_t st) { cudaError_t e = alloc(count); if (e != cudaSuccess || !count) return e; return cudaMemcpyAsync(p, src, count * sizeof(T), cudaMemcpyHostToDevice, st); }
};

inline double median_like_reference(std::vector<double> v) {   // utils::MedianOfDoubleVec (src/utils/utils.cc:77-97)
  const size_t n = v.size();
  if (n % 2 == 0) {
    std::nth_element(v.begin(), v.begin() + n / 2 - 1, v.end()); const double e1 = v[n / 2 - 1];
    std::nth_element(v.begin(), v.begin() + n / 2, v.end()); const double e2 = v[n / 2];
    return (e1 + e2) / 2;
  }
  std::nth_element(v.begin(), v.begin() + n / 2, v.end());
  return v[n / 2];
}

// CSR by board point of the corners selected by `take(c)`: pt_off[np + 1], pt_obs[...] (counting sort, stable in corner order)
template <class F>
void build_point_adjacency(int np, int nc, const int32_t* ids, F take, std::vector<int>& pt_off, std::vector<int>& pt_obs) {
  pt_off.assign(np + 1, 0);
  for (int c = 0; c < nc; ++c) if (take(c)) ++pt_off[ids[c] + 1];
  for (int p = 0; p < np; ++p) pt_off[p + 1] += pt_off[p];
  pt_obs.resize(pt_off[np]);
  std::vector<int> fill(pt_off.begin(), pt_off.end() - 1);
  for (int c = 0; c < nc; ++c) if (take(c)) pt_obs[fill[ids[c]]++] = c;
}

// ---- icc_pose.cu: the board, the corner CSR of nf views (off[nf + 1], checked by the caller) and the pose kernels' work buffers ----
struct BoardViews {
  int nf = 0, nc = 0, np = 0;
  DevBuf<double4> board; DevBuf<double2> uv, xy; DevBuf<int> off, pid, ok, valid; DevBuf<unsigned char> use; DevBuf<double> q, p, e;
  DevBuf<double4> bear; DevBuf<int> okh;   // tangent mode only: corner bearings, and the start's per-corner flags
};
icc_status upload_board_views(cudaStream_t st, int np, const double* points, int nf, const int32_t* off, const int32_t* ids, const double* uv, BoardViews& B, std::string& err);
// the poses, mean errors (optional) and valid flags of B's views to the host; waits for the stream
icc_status read_poses(cudaStream_t st, const BoardViews& B, double* q_wc, double* p_wc, double* mean_err, int32_t* valid, std::string& err);
// theia::BundleAdjustTracks with constant cameras: Q carries the camera, measurements, poses and board_in; corner c observes point ids[c]
// from view obs_view[c] and takes part iff obs_view[c] >= 0.  Refined points -> d_out and points_out (4 doubles each).  With bear (the corners'
// bearings) the residual is the tangent error and Q.meas is not read.  With rs every corner is seen at its row time (the pose step's rolling shutter).
icc_status refine_board_points(cudaStream_t st, PointProblem Q, int nc, const int32_t* ids, const std::vector<int>& obs_view, DevBuf<double4>& d_out, std::vector<double>& points_out, int& n_opt, std::string& err,
                               const double4* bear = nullptr, const RsPass* rs = nullptr);

// ---- the upstream tools' host drivers, each in the .cu file of its kernels -----------------------------------------------------
icc_status pixels_to_normalized(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int n, const double* uv, double* xy_out, int32_t* ok, std::string& err);
icc_status pixels_to_bearings(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int n, const double* uv, double* xyz_out, int32_t* ok, std::string& err);
// pose_error: ICC_POSE_ERROR_NORMALIZED or ICC_POSE_ERROR_TANGENT (the residual of the per-view refinement and of the board points)
// The shutter of the pose step (icc_set_pose_rolling_shutter): line_delay = 0 is the global shutter; otherwise frame_t holds the nf view times,
// and vel (6 per view: w, u) and n_static (valid views without a neighbour in time) receive what the last rolling-shutter pass used.
struct PoseShutter { double line_delay = 0.0; const double* frame_t = nullptr; double* vel = nullptr; int32_t* n_static = nullptr; };
icc_status estimate_board_poses(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int W, int H, int np, const double* points, int nf, const int32_t* off,
                                const int32_t* ids, const double* uv, double max_reproj_error, int min_points, int pose_error, const PoseShutter& shutter, double* q_wc, double* p_wc, double* mean_err,
                                int32_t* valid, std::string& err);
icc_status optimize_board_points(cudaStream_t st, int model, const double intr[ICC_MAX_INTRINSICS], int W, int H, int np, const double* points, int nf, const int32_t* off, const int32_t* ids,
                                 const double* uv, double max_reproj_error, int min_points, int min_observations, int pose_error, const PoseShutter& shutter, double* q_wc, double* p_wc,
                                 double* mean_err, int32_t* valid, std::vector<double>& points_out, int32_t* n_opt_out, std::string& err);
void filter_bad_poses(int nv, const double* p_wc, int32_t* valid);
icc_status estimate_imu_to_camera_rotation(cudaStream_t st, int sm_count, int n_views, const double* view_t, const double* q_cw, int n_imu, const double* imu_t, const double* gyro,
                                           const double* bias_in, double* q_out, double* td_out, double* bias_out, double* err_out, int32_t* iters_out, std::string& err);
icc_status spline_error_weighting(cudaStream_t st, int sm_count, int n, const double* times, const double* signal, double quality, double min_dt, double max_dt, double* dt_out, double* var_out, double* spectrum, std::string& err);
icc_status imu_biases(cudaStream_t st, int sm_count, int n, const double* acc, const double* gyr, double gravity_const, double accl_bias[3], double gyro_bias[3], std::string& err);
// The shutter of the camera calibration (icc_set_camcal_rolling_shutter): line_delay = 0 is the global shutter; otherwise vel holds the fixed
// camera-frame velocities (w, u) of the nv views, 6 doubles each, and corner c is seen uv[c].y * line_delay after its frame.
struct CamCalShutter { double line_delay = 0.0; const double* vel = nullptr; };
// S.success = 0 when too few views remain; with optimize_board_points the refined board comes back in points_out (empty otherwise)
icc_status calibrate_camera(cudaStream_t st, int model, int W, int H, int np, const double* points, int nv, const int32_t* off, const int32_t* ids, const double* uv,
                            const double* q_init, const double* p_init, const int32_t* init_valid, double focal_init, double distortion_init, const icc_camcal_options* options,
                            double* intr_out, double* q_out, double* p_out, double* err_out, int32_t* used_out, icc_camcal_summary& S, std::vector<double>& points_out, std::string& err,
                            const CamCalShutter& shutter = CamCalShutter{});
void default_static_imu_options(icc_static_imu_options* o);
icc_status static_imu_calibrate(cudaStream_t st, int n, const double* t, const double* acc, const double* gyr, const icc_static_imu_options& o,
                                double acc_out[9], double gyr_out[9], double bias_out[3], icc_static_imu_summary& S, std::vector<int32_t>& intervals, std::string& err);
namespace allan { struct Curves; }   // icc_allan_math.cuh
void default_allan_options(icc_allan_options* o);
icc_status allan_variance(cudaStream_t st, int n, const double* t, const double* acc, const double* gyr, const icc_allan_options& o,
                          double params[30], icc_allan_noise noise[6], icc_allan_summary summary[6], allan::Curves& curves, std::string& err);
// bgr: rows hold width interleaved B, G, R bytes (icc_extract_radon_board_bgr); else width gray bytes
icc_status extract_radon_board(cudaStream_t st, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, bool frames_on_device, bool bgr, int W, int H,
                               double f, double* uv_out, int32_t* found, icc_board_summary& S, std::string& err);

// 8-bit gray frames; uv_out / status_out per frame and point id (icc_extract_aprilgrid)
icc_status extract_aprilgrid(cudaStream_t st, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, bool frames_on_device, int tags_x, int tags_y,
                             double f, double* uv_out, int32_t* status_out, int32_t* found, icc_aprilgrid_summary& S, std::string& err);
}  // namespace icc
