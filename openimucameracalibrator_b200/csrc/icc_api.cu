// C-ABI + host logic of the H100 calibration solver (see include/icc_b200.h for the boundary contract).
//
// Host side mirrors, in its own structure, what the reference does on one thread before/around ceres::Solve:
//   ImuCameraCalibrator::BatchInitSpline / InitializeGravity / Optimize   src/core/imu_camera_calibrator.cc:21-168
//   SplineTrajectoryEstimator::SetTimes / InitBiasSplines / BatchInitSO3R3VisPoses / Add*Measurement / CalcTimes /
//   SetFixedParams / Optimize / getters       include/OpenCameraCalibrator/core/spline_trajectory_estimator.impl.h
//   InterpolateQuaternions / InterpolateVector3d                           src/utils/utils.cc:194-261
// Everything numerical per LM iteration runs on the GPU (icc_eval.cu, icc_solver.cu); the host only sequences launches
// and applies the trust-region accept/reject logic to a few scalars read back per iteration.  There is no CPU fallback.
#include "../../include/icc_b200.h"
#include "icc_allan_math.cuh"
#include "icc_bias_prior.cuh"
#include "icc_bearing_math.cuh"
#include "icc_camera.cuh"
#include "icc_host.h"
#include "icc_rotinit_math.cuh"
#include "icc_trust_region.cuh"
#include "icc_vision_rows.cuh"

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

using namespace icc;


namespace {

constexpr double S_TO_NS = 1e9;

// Host staging of the large measurement arrays (corners, IMU samples): page-locked blocks from a process-wide cache (the first
// job pays cudaHostAlloc, later ones reuse), so that the uploads of BatchInitSpline are asynchronous DMA transfers that overlap the
// host assembly.  Host-only handles (and a failed cudaHostAlloc) use ordinary memory; the copies then stage through the driver.
struct PinnedCache {
  std::mutex mu;
  std::multimap<size_t, void*> free_blocks;
  void* get(size_t bytes, size_t* cap) {
    {
      std::lock_guard<std::mutex> lk(mu);
      auto it = free_blocks.lower_bound(bytes);
      if (it != free_blocks.end() && it->first <= 2 * bytes + 4096) { void* q = it->second; *cap = it->first; free_blocks.erase(it); return q; }
    }
    void* q = nullptr;
    if (cudaHostAlloc(&q, bytes, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    *cap = bytes; return q;
  }
  void put(size_t bytes, void* q) { std::lock_guard<std::mutex> lk(mu); free_blocks.emplace(bytes, q); }
  void trim() { std::lock_guard<std::mutex> lk(mu); for (auto& kv : free_blocks) cudaFreeHost(kv.second); free_blocks.clear(); }
};
PinnedCache& pinned_cache() { static PinnedCache* c = new PinnedCache(); return *c; }

template <class T>
struct HostBuf {
  T* p = nullptr; size_t n = 0, cap_bytes = 0; bool pinned = false;
  HostBuf() = default; HostBuf(const HostBuf&) = delete; HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() { release(); }
  void release() { if (p) { if (pinned) pinned_cache().put(cap_bytes, p); else free(p); } p = nullptr; n = 0; cap_bytes = 0; pinned = false; }
  void resize(size_t count, bool want_pinned) {    // contents are NOT preserved
    const size_t bytes = std::max<size_t>(256, (count * sizeof(T) + 255) / 256 * 256);
    if (!(p && cap_bytes >= bytes && (pinned || !want_pinned))) {
      release();
      if (want_pinned) { size_t cap = 0; p = static_cast<T*>(pinned_cache().get(bytes, &cap)); if (p) { pinned = true; cap_bytes = cap; } }
      if (!p) { p = static_cast<T*>(malloc(bytes)); cap_bytes = bytes; pinned = false; }
    }
    n = count;
  }
  void assign(const T* src, size_t count, bool want_pinned) { resize(count, want_pinned); if (count) memcpy(p, src, count * sizeof(T)); }   // (splitting this copy over threads was measured: the later DMA / reads get slower by more than the copy gains)
  void clear() { n = 0; }
  T* data() { return p; } const T* data() const { return p; }
  size_t size() const { return n; } bool empty() const { return n == 0; }
  T& operator[](size_t i) { return p[i]; } const T& operator[](size_t i) const { return p[i]; }
  const T* begin() const { return p; } const T* end() const { return p + n; }
};

// Bump allocator over one page-locked block: the many small arrays a job uploads (frame tables, work lists, knots) are staged here
// and copied asynchronously, instead of one blocking pageable cudaMemcpy each.  reset() only after the stream has drained.
struct PinnedArena {
  HostBuf<unsigned char> buf; size_t used = 0;
  void reset(size_t capacity, bool pin) { if (buf.size() < capacity) buf.resize(capacity, pin); used = 0; }
  void* take(size_t bytes) { const size_t o = (used + 255) & ~size_t(255); if (o + bytes > buf.size()) return nullptr; used = o + bytes; return buf.data() + o; }
};

struct StateBufs {
  DevBuf<double4> so3, r3, ba, bg; DevBuf<double> glob;
  DevBuf<double4> pts, board; DevBuf<double> pjac;   // board points of the state (icc_points.cu)
  DeviceState view() const { DeviceState s; s.so3 = so3.p; s.r3 = r3.p; s.ba = ba.p; s.bg = bg.p; s.glob = glob.p; s.pts = pts.p; s.board = board.p; s.pjac = pjac.p; return s; }
};

struct FrameHost { double t_s; int c0, c1; int s_so3, s_r3; double u_so3, u_r3; };

}  // namespace

struct icc_handle {
  std::string err = "";
  int device = -1;
  icc_solver_options opt;
  // ---- raw inputs -------------------------------------------------------------------------------------------
  int model = -1, n_intr = 0, width = 0, height = 0; double intr[MAX_INTR] = {0};
  int pose_error = ICC_POSE_ERROR_NORMALIZED;   // residual of icc_estimate_board_poses / icc_optimize_board_points (icc_set_pose_error)
  int reproj_error = ICC_REPROJ_ERROR_PIXEL;     // vision residual of the spline solve (icc_set_reprojection_error), fixed at batch_init
  double pose_line_delay = 0.0; std::vector<double> pose_frame_t;   // their shutter (icc_set_pose_rolling_shutter; 0 = global)
  std::vector<double> pose_vel; int32_t pose_n_static = 0;          // what their last rolling-shutter pass used (icc_get_pose_velocities)
  double camcal_line_delay = 0.0; std::vector<double> camcal_frame_t, camcal_w_u;   // shutter of icc_calibrate_camera (icc_set_camcal_rolling_shutter)
  int32_t camcal_n_views = 0;
  std::vector<double> camcal_vel; int32_t camcal_n_static = 0;      // what its last rolling-shutter calibration used (icc_get_camcal_velocities)
  std::vector<double> points;
  std::vector<double> frame_t; std::vector<int> corner_off; HostBuf<int> point_ids; HostBuf<double> uv; std::vector<double> q_wc, p_wc;
  HostBuf<double> imu_t, imu_acc, imu_gyr;
  int id_lo = 0, id_hi = -1;                 // range of the corner point ids (found while set_frames copies them)
  // Page-locked caller buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory): set_frames / set_imu send the big arrays straight to the
  // device by DMA and wait for it, instead of staging them through a host copy first; the host then only keeps what it reads (time stamps,
  // offsets, poses) and fetches the rest back from the device in the rare paths that gather (unsorted streams, non-contiguous shards).
  bool frames_dev = false, imu_dev = false; size_t n_corners_in = 0, n_imu_in = 0;
  bool imu_sorted = false;                   // imu_t is non-decreasing (found while set_imu copies it)
  int shard_rank = 0, shard_world = 1;
  icc_allreduce_fn allreduce = nullptr; void* allreduce_user = nullptr;
  icc_comm* comm = nullptr;                  // borrowed NCCL communicator (icc_set_comm): the native cross-rank sum
  // ---- assembled problem (host) -----------------------------------------------------------------------------
  bool initialised = false;
  icc_init_params ip;
  int64_t dt_so3_ns = 0, dt_r3_ns = 0, dt_ba_ns = 0, dt_bg_ns = 0, start_ns = 0, end_ns = 0;
  // bias splines: spacing [s] of icc_set_bias_splines (<= 0: the reference's 10 s) and the random-walk densities of icc_set_bias_random_walk
  // (walk_set[s] = false: no prior rows), both read by the next icc_batch_init_spline into `prior` (0 = accelerometer, 1 = gyroscope)
  double bias_dt_s_set[2] = {0.0, 0.0}; bool walk_set[2] = {false, false}; double walk_q_set[2][3] = {{0.0}};
  BiasPrior prior{};        // the prior of the assembled problem (on[s] only on shard 0, which owns the rows)
  int n_res_prior = 0;      // its rows in this shard
  double t0_s = 0, tend_s = 0, max_ba = 1.0, max_bg = 0.1;
  std::vector<double> so3, r3, ba, bg;       // host mirror of the state (4/3/3/3 doubles per knot)
  double glob[G_COUNT] = {0};
  std::vector<FrameHost> frames;             // frames in the problem (this shard)
  std::vector<double> used_uv; std::vector<int> used_pid;   // gathered corners -- only when the used frames are not one contiguous run
  bool used_contig = false; int used_c0 = 0, used_n = 0;    // ... otherwise corners [used_c0, used_c0 + used_n) of uv / point_ids are used in place
  bool imu_contig = false; int imu_src0 = 0;                // same for the accelerometer / gyroscope samples
  std::vector<std::pair<int, int>> frame_in;               // input corner range (icc_set_frames) of every frame in the problem
  size_t n_corners_assembled = 0;                           // corners given to icc_set_frames when the problem was assembled
  bool corners_rejected = false;                            // icc_reject_outlier_corners has compacted the corners since batch_init
  std::vector<double> imu_used_t, imu_used_acc, imu_used_gyr; HostBuf<int64_t> imu_used_st;
  size_t n_imu_used = 0;                     // kept samples; imu_used_t / imu_used_st are only materialised off the sorted fast path (imu_lazy == false)
  bool imu_lazy = false;                     // sorted fast path: kept samples = imu_t[imu_src0 .. +n_imu_used) + time offset, relative times derived on the device
  std::vector<ImuCell> cells;
  int dropped_frames = 0, dropped_imu = 0;
  // ---- device ---------------------------------------------------------------------------------------------------
  cudaStream_t stream = nullptr;
  EvalAux aux{};            // second stream + fork/join events: vision and IMU kernels of one evaluation run concurrently
  bool aux_ok = false;
  int sm_count = 132;
  StateBufs st[2]; int cur = 0;
  HostBuf<unsigned char> small_pinned; DevBuf<int> d_idrange;
  void* arena_small(size_t bytes) { if (small_pinned.size() < bytes) small_pinned.resize(std::max<size_t>(bytes, 256), true); return small_pinned.pinned ? small_pinned.data() : nullptr; }
  DevBuf<double2> d_uv_all; DevBuf<int> d_pid_all; DevBuf<double> d_acc_all, d_gyr_all;   // complete input arrays (frames_dev / imu_dev)
  DevBuf<double4> d_board; DevBuf<int> d_f_off, d_f_s_so3, d_f_s_r3, d_pid; DevBuf<double> d_f_u_so3, d_f_u_r3; DevBuf<double2> d_uv;
  DevBuf<double> d_view_t, d_view_q, d_view_p;   // per-view pose priors in time order (knot initialisation kernel)
  DevBuf<VisFrame> d_vframes; DevBuf<VisItem> d_vitems;
  DevBuf<double4> d_bear; DevBuf<int> d_bear_ok;   // tangent mode: the used corners' bearings, in stream order next to P.uv
  // outlier corners: residual pairs, errors and sums of the error pass; input index of every corner (once rejected); compaction targets
  DevBuf<double> d_cres, d_cerr, d_osum; DevBuf<int> d_csrc, d_ckept, d_in_off, d_foff_new;
  DevBuf<double2> d_uv_new; DevBuf<int> d_pid_new, d_bear_ok_new, d_csrc_new; DevBuf<double4> d_bear_new;
  TangentMeas tan{nullptr, nullptr, 0.0};          // ... and what the evaluation kernels read of them (tangent_meas)
  DevBuf<ImuCellP> d_icells; DevBuf<VisItem> d_iitems;
  std::vector<VisItem> vitems, iitems;   // host copies of the per-warp runs (icc_get_eval_schedule)
  DevBuf<double> d_imu_traw; DevBuf<VisionWork> d_vwork; DevBuf<int64_t> d_imu_t; DevBuf<double> d_imu_acc, d_imu_gyr; DevBuf<ImuCell> d_cells, d_iwork;
  DevBuf<int> d_so3_col, d_r3_col, d_ba_col, d_bg_col;
  DevBuf<double> d_incr;     // SO(3) increment table of the persistent Jacobian evaluation (DeviceProblem::incr)
  DevBuf<double> d_ne, d_scale, d_ws, d_delta, d_scal, d_res;
  PinnedArena arena;        // staging of the small uploads of BatchInitSpline
  DeviceProblem P;
  bool state_dirty_host = false;   // device state newer than host mirror
  bool glob_host_current = false;  // ... but the small block of globals (T_i_c, gravity, line delay, intrinsics) was already read back
  bool knots_dirty_host = false;   // only the spline knots are newer on the device (device-side initialisation): globals / biases on the host are current
  // ---- active set ------------------------------------------------------------------------------------------------
  int cur_flags = -1;
  int ne_flags = -1;        // flags of the normal equations in d_ne that icc_evaluate / icc_normal_matvec left for icc_solve_normal_equations (-1: none)
  std::vector<int> so3_col, r3_col, ba_col, bg_col;   // solver index of first dim or -1
  int col_tic = -1, col_g = -1, col_ld = -1;
  int n_tan = 0;
  std::vector<int> perm;           // canonical tangent index -> solver index
  int launches_at_start = 0;
  std::vector<int32_t> static_imu_intervals;   // kept static intervals of the last icc_static_imu_calibration
  allan::Curves allan_curves;                  // curves of the last icc_allan_variance
};

namespace {

icc_status fail(icc_handle* h, icc_status s, const std::string& m) { if (h) h->err = m; return s; }
// ICC_TRACE_PHASES=1: host wall clock between the marked points of a call, to stderr (diagnosis only; synchronises the stream at every mark)
struct PhaseTrace {
  bool on; cudaStream_t st; std::chrono::steady_clock::time_point t;
  PhaseTrace(cudaStream_t s) : on(getenv("ICC_TRACE_PHASES") != nullptr), st(s), t(std::chrono::steady_clock::now()) {}
  void lap(const char* what) {
    if (!on) return;
    const auto a = std::chrono::steady_clock::now(); if (st) cudaStreamSynchronize(st); const auto b = std::chrono::steady_clock::now();
    fprintf(stderr, "[icc phase] %-28s %8.3f ms host + %7.3f ms stream drain\n", what, std::chrono::duration<double, std::milli>(a - t).count(), std::chrono::duration<double, std::milli>(b - a).count());
    t = std::chrono::steady_clock::now();
  }
};
#define CU(call) ICC_CUDA_CHECK(call, h->err)
#define NEED_DEVICE() do { if (h->device < 0) return fail(h, ICC_ERR_NO_DEVICE, "no CUDA device bound to this handle (host-only handle): compute entry points are unavailable"); } while (0)
// Runs an upstream tool's host driver (icc_host.h) on the handle's device; a failed driver's message becomes the handle's error.
template <class F> icc_status drive(icc_handle* h, F driver) {
  CU(cudaSetDevice(h->device));
  std::string err;
  const icc_status rc = driver(err);
  return rc == ICC_OK ? rc : fail(h, rc, err);
}

Q4 qn(const double* q) { return qnormalized(q4(q[0], q[1], q[2], q[3])); }

// CalcTimes (impl.h:763-788)
bool calc_times(int64_t sensor_ns, int64_t start_ns, int64_t dt_ns, size_t nr_knots, int N, double& u, int64_t& s) {
  const int64_t st = sensor_ns - start_ns;
  if (st < 0) { u = 0.0; return false; }
  s = st / dt_ns;
  if (s < 0) return false;
  if (size_t(s + N) > nr_knots) return false;
  u = double(st % dt_ns) / double(dt_ns);
  return true;
}

Pose pose_inv(const Pose& a) { const Q4 qi = qnormalized(qconj(a.q)); return {qi, qrot(qi, -a.t)}; }

std::vector<double4> pad4(const std::vector<double>& v, int dim) {
  const size_t n = v.size() / dim; std::vector<double4> o(n);
  for (size_t i = 0; i < n; ++i) o[i] = make_double4(v[dim * i], v[dim * i + 1], v[dim * i + 2], dim == 4 ? v[dim * i + 3] : 0.0);
  return o;
}

// v -> d through the handle's staging arena (asynchronous on the handle's stream); falls back to the blocking copy when the arena is full
template <class T>
cudaError_t upload_staged(icc_handle* h, DevBuf<T>& d, const std::vector<T>& v) {
  cudaError_t e = d.alloc(v.size()); if (e != cudaSuccess || v.empty()) return e;
  const size_t bytes = v.size() * sizeof(T);
  void* stage = h->arena.take(bytes);
  if (!stage) return cudaMemcpy(d.p, v.data(), bytes, cudaMemcpyHostToDevice);
  memcpy(stage, v.data(), bytes);
  return cudaMemcpyAsync(d.p, stage, bytes, cudaMemcpyHostToDevice, h->stream);
}

// board points of state `which`: homogeneous vectors up, de-homogenised copy + local Jacobians derived on the device
icc_status upload_points(icc_handle* h, int which, bool staged) {
  h->ne_flags = -1;                        // every state upload passes here: the normal equations no longer belong to the state
  StateBufs& s = h->st[which];
  const size_t np = h->points.size() / 4;
  if (!np) return ICC_OK;
  CU(s.board.alloc(np)); CU(s.pjac.alloc(12 * np));
  if (staged) { CU(upload_staged(h, s.pts, pad4(h->points, 4))); }
  else { CU(cudaStreamSynchronize(h->stream)); CU(s.pts.upload(pad4(h->points, 4))); }
  launch_points_prepare((int)np, s.pts.p, s.board.p, s.pjac.p, h->stream);
  if (!staged) CU(cudaStreamSynchronize(h->stream));
  return ICC_OK;
}

bool host_is_pinned(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}
// host copies of the arrays that went straight to the device, for the paths that gather on the host
icc_status ensure_host_corners(icc_handle* h) {
  if (!h->frames_dev || h->uv.size() == 2 * h->n_corners_in) return ICC_OK;
  h->uv.resize(2 * h->n_corners_in, true); h->point_ids.resize(h->n_corners_in, true);
  CU(cudaStreamSynchronize(h->stream));
  if (h->n_corners_in) { CU(cudaMemcpy(h->uv.data(), h->d_uv_all.p, h->n_corners_in * sizeof(double2), cudaMemcpyDeviceToHost)); CU(cudaMemcpy(h->point_ids.data(), h->d_pid_all.p, h->n_corners_in * sizeof(int), cudaMemcpyDeviceToHost)); }
  return ICC_OK;
}
icc_status ensure_host_imu(icc_handle* h) {
  if (!h->imu_dev || h->imu_acc.size() == 3 * h->n_imu_in) return ICC_OK;
  h->imu_acc.resize(3 * h->n_imu_in, true); h->imu_gyr.resize(3 * h->n_imu_in, true);
  CU(cudaStreamSynchronize(h->stream));
  if (h->n_imu_in) { CU(cudaMemcpy(h->imu_acc.data(), h->d_acc_all.p, 3 * h->n_imu_in * sizeof(double), cudaMemcpyDeviceToHost)); CU(cudaMemcpy(h->imu_gyr.data(), h->d_gyr_all.p, 3 * h->n_imu_in * sizeof(double), cudaMemcpyDeviceToHost)); }
  return ICC_OK;
}

icc_status upload_state(icc_handle* h, int which, bool staged = false) {
  StateBufs& s = h->st[which];
  std::vector<double> g(h->glob, h->glob + G_COUNT);
  { icc_status r = upload_points(h, which, staged); if (r != ICC_OK) return r; }
  if (staged) {
    CU(upload_staged(h, s.so3, pad4(h->so3, 4))); CU(upload_staged(h, s.r3, pad4(h->r3, 3))); CU(upload_staged(h, s.ba, pad4(h->ba, 3))); CU(upload_staged(h, s.bg, pad4(h->bg, 3)));
    CU(upload_staged(h, s.glob, g));
    return ICC_OK;
  }
  CU(cudaStreamSynchronize(h->stream));   // a staged upload of the same buffers may still be in flight
  CU(s.so3.upload(pad4(h->so3, 4))); CU(s.r3.upload(pad4(h->r3, 3))); CU(s.ba.upload(pad4(h->ba, 3))); CU(s.bg.upload(pad4(h->bg, 3)));
  CU(s.glob.upload(g));
  return ICC_OK;
}

icc_status sync_state_to_host(icc_handle* h) {
  if (!(h->state_dirty_host || h->knots_dirty_host) || h->device < 0) return ICC_OK;
  const StateBufs& s = h->st[h->cur];
  auto pull = [&](const DevBuf<double4>& d, std::vector<double>& v, int dim) -> cudaError_t {
    std::vector<double4> tmp(d.n);
    if (d.n) { cudaError_t e = cudaMemcpy(tmp.data(), d.p, d.n * sizeof(double4), cudaMemcpyDeviceToHost); if (e != cudaSuccess) return e; }
    for (size_t i = 0; i < d.n; ++i) { v[dim * i] = tmp[i].x; v[dim * i + 1] = tmp[i].y; v[dim * i + 2] = tmp[i].z; if (dim == 4) v[dim * i + 3] = tmp[i].w; }
    return cudaSuccess;
  };
  CU(cudaStreamSynchronize(h->stream));
  CU(pull(s.so3, h->so3, 4)); CU(pull(s.r3, h->r3, 3)); CU(pull(s.ba, h->ba, 3)); CU(pull(s.bg, h->bg, 3));
  CU(cudaMemcpy(h->glob, s.glob.p, G_COUNT * sizeof(double), cudaMemcpyDeviceToHost));
  if (h->state_dirty_host && s.pts.n * 4 == h->points.size()) CU(pull(s.pts, h->points, 4));
  h->state_dirty_host = false; h->knots_dirty_host = false;
  return ICC_OK;
}

// getters of the globals (T_i_c, gravity, line delay, ...) after a solve: 25 doubles instead of every knot
icc_status sync_globals_to_host(icc_handle* h) {
  if (!h->state_dirty_host || h->glob_host_current || h->device < 0) return ICC_OK;
  CU(cudaMemcpyAsync(h->glob, h->st[h->cur].glob.p, G_COUNT * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  h->glob_host_current = true;
  return ICC_OK;
}

icc_status push_state_to_device(icc_handle* h) {
  if (h->device < 0 || !h->initialised) return ICC_OK;
  icc_status s = upload_state(h, h->cur);
  h->state_dirty_host = false; h->knots_dirty_host = false;
  return s;
}

// Active set (SetFixedParams, impl.h:92-252) -> column maps in SOLVER order: spline knots sorted by knot time (SO3 before
// R3 on ties) form the banded part; T_i_c, gravity, line delay and bias knots form the border.
icc_status configure(icc_handle* h, int flags) {
  if ((flags & ICC_FLAG_POINTS) && (flags & ICC_FLAG_CAM_INTRINSICS)) return fail(h, ICC_ERR_UNSUPPORTED, "POINTS together with CAM_INTRINSICS (an extension flag of this library) is not supported");
  if (h->reproj_error == ICC_REPROJ_ERROR_TANGENT && (flags & ICC_FLAG_CAM_INTRINSICS))
    return fail(h, ICC_ERR_UNSUPPORTED, "CAM_INTRINSICS with the tangent reprojection error is not supported: the corners' bearings are fixed by the intrinsics at batch_init_spline");
  if (h->cur_flags == flags) return ICC_OK;
  // the host layout below is rewritten before the shape checks: until it is complete, no flags are configured, so that a refused
  // shape cannot leave its layout behind under the previous flags (the device-side problem P keeps the previous layout, complete)
  h->cur_flags = -1; h->ne_flags = -1;
  const int nso3 = (int)h->so3.size() / 4, nr3 = (int)h->r3.size() / 3, nba = (int)h->ba.size() / 3, nbg = (int)h->bg.size() / 3;
  const bool spline = flags & ICC_FLAG_SPLINE, tic = flags & ICC_FLAG_T_I_C, grav = flags & ICC_FLAG_GRAVITY_DIR;
  const bool ld = (flags & ICC_FLAG_CAM_LINE_DELAY) && h->ip.init_line_delay_s != 0.0;
  const bool ab = flags & (ICC_FLAG_ACC_BIAS | ICC_FLAG_IMU_BIASES), gb = flags & (ICC_FLAG_GYR_BIAS | ICC_FLAG_IMU_BIASES);
  const bool intr = flags & ICC_FLAG_IMU_INTRINSICS, cam_intr = flags & ICC_FLAG_CAM_INTRINSICS, toff = flags & ICC_FLAG_TIME_OFFSET;
  const int npts = (int)(h->points.size() / 4);
  const bool pts = (flags & ICC_FLAG_POINTS) && npts > 0;      // every track a view sees (impl.h:136-152); points no view sees get zero columns
  // canonical offsets
  int n = 0;
  const int c_so3 = spline ? n : -1; if (spline) n += 3 * nso3;
  const int c_r3 = spline ? n : -1; if (spline) n += 3 * nr3;
  const int c_tic = tic ? n : -1; if (tic) n += 6;
  const int c_g = grav ? n : -1; if (grav) n += 3;
  const int c_ld = ld ? n : -1; if (ld) n += 1;
  const int c_ba = ab ? n : -1; if (ab) n += 3 * nba;
  const int c_bg = gb ? n : -1; if (gb) n += 3 * nbg;
  const int c_ai = intr ? n : -1; if (intr) n += 6;
  const int c_gi = intr ? n : -1; if (intr) n += 9;
  const int c_ci = cam_intr ? n : -1; if (cam_intr) n += h->n_intr;
  const int c_to = toff ? n : -1; if (toff) n += 1;
  const int c_pts = pts ? n : -1; if (pts) n += 3 * npts;
  h->n_tan = n;
  h->so3_col.assign(nso3, -1); h->r3_col.assign(nr3, -1); h->ba_col.assign(nba, -1); h->bg_col.assign(nbg, -1);
  int pos = 0;
  if (spline) {
    int i = 0, j = 0;
    while (i < nso3 || j < nr3) {
      const bool take_so3 = j >= nr3 || (i < nso3 && int64_t(i) * h->dt_so3_ns <= int64_t(j) * h->dt_r3_ns);
      if (take_so3) h->so3_col[i++] = pos; else h->r3_col[j++] = pos;
      pos += 3;
    }
  }
  const int nk = pos;
  h->col_tic = tic ? pos : -1; if (tic) pos += 6;
  h->col_g = grav ? pos : -1; if (grav) pos += 3;
  h->col_ld = ld ? pos : -1; if (ld) pos += 1;
  if (ab) for (int k = 0; k < nba; ++k) { h->ba_col[k] = pos; pos += 3; }
  if (gb) for (int k = 0; k < nbg; ++k) { h->bg_col[k] = pos; pos += 3; }
  const int col_ai = intr ? pos : -1; if (intr) pos += 6;
  const int col_gi = intr ? pos : -1; if (intr) pos += 9;
  const int col_ci = cam_intr ? pos : -1; if (cam_intr) pos += h->n_intr;
  const int col_to = toff ? pos : -1; if (toff) pos += 1;
  const int col_pts = pts ? pos : -1; if (pts) pos += 3 * npts;
  const int nb = pos - nk;
  h->perm.assign(n, -1);
  if (spline) { for (int k = 0; k < nso3; ++k) for (int d = 0; d < 3; ++d) h->perm[c_so3 + 3 * k + d] = h->so3_col[k] + d; for (int k = 0; k < nr3; ++k) for (int d = 0; d < 3; ++d) h->perm[c_r3 + 3 * k + d] = h->r3_col[k] + d; }
  if (tic) for (int d = 0; d < 6; ++d) h->perm[c_tic + d] = h->col_tic + d;
  if (grav) for (int d = 0; d < 3; ++d) h->perm[c_g + d] = h->col_g + d;
  if (ld) h->perm[c_ld] = h->col_ld;
  if (ab) for (int k = 0; k < nba; ++k) for (int d = 0; d < 3; ++d) h->perm[c_ba + 3 * k + d] = h->ba_col[k] + d;
  if (gb) for (int k = 0; k < nbg; ++k) for (int d = 0; d < 3; ++d) h->perm[c_bg + 3 * k + d] = h->bg_col[k] + d;
  if (intr) { for (int d = 0; d < 6; ++d) h->perm[c_ai + d] = col_ai + d; for (int d = 0; d < 9; ++d) h->perm[c_gi + d] = col_gi + d; }
  if (cam_intr) for (int d = 0; d < h->n_intr; ++d) h->perm[c_ci + d] = col_ci + d;
  if (toff) h->perm[c_to] = col_to;
  if (pts) for (int d = 0; d < 3 * npts; ++d) h->perm[c_pts + d] = col_pts + d;
  // half bandwidth: widest knot window touched by one residual block
  int kd = 0;
  if (spline) {
    auto span = [&](int s_so3, int s_r3, bool use_r3) {
      int lo = h->so3_col[s_so3], hi = h->so3_col[s_so3 + SPLINE_N - 1] + 2;
      if (use_r3) { lo = std::min(lo, h->r3_col[s_r3]); hi = std::max(hi, h->r3_col[s_r3 + SPLINE_N - 1] + 2); }
      kd = std::max(kd, hi - lo);
    };
    if (h->ip.init_line_delay_s != 0.0) for (const auto& f : h->frames) span(f.s_so3, f.s_r3, true);
    for (const auto& c : h->cells) span(c.s_so3, c.s_r3, true);
    if (h->shard_world > 1) {   // every rank must agree on the layout: use the global worst case of the time-sorted order
      for (int s = 0; s + SPLINE_N <= nso3; ++s) { const int64_t t = int64_t(s) * h->dt_so3_ns; const int sr = (int)std::min<int64_t>(t / h->dt_r3_ns, nr3 - SPLINE_N); span(s, sr, true); }
      for (int s = 0; s + SPLINE_N <= nr3; ++s) { const int64_t t = int64_t(s) * h->dt_r3_ns; const int ss = (int)std::min<int64_t>(t / h->dt_so3_ns, nso3 - SPLINE_N); span(ss, s, true); }
    }
  }
  if (kd > 255) return fail(h, ICC_ERR_UNSUPPORTED, "knot-spacing ratio produces a half bandwidth > 255");
  {   // the knot band alone must fit an elimination plan; a border that does not fit is reported by the solve (evaluation works at any width)
    DeviceProblem B; memset(&B, 0, sizeof B);
    B.nk = nk; B.kd = kd; B.ldb = kd + 1;
    icc_solver_plan_info pi; solver_plan_info(B, 0, &pi);
    if (!pi.valid) {
      // a band too wide for several chunks leaves one chunk, whose back-substitution holds every knot column in shared memory:
      // find the longest sequence that one chunk of this band takes (none from a half bandwidth of 112: the level-0 window alone is too large)
      int lo = 0, hi = nk;
      while (lo < hi) { const int mid = lo + (hi - lo + 1) / 2; B.nk = mid; solver_plan_info(B, 1, &pi); if (pi.valid) lo = mid; else hi = mid - 1; }
      char msg[400];
      if (lo > 0)
        snprintf(msg, sizeof msg, "the knot spacing (dt_so3 / dt_r3 ratio) gives a half bandwidth of %d columns over %d knot columns: no elimination "
                 "plan of the solver fits in shared memory (a band this wide is solved as one chunk, which takes at most %d knot columns; "
                 "use a knot-spacing ratio closer to 1 or a shorter sequence)", kd, nk, lo);
      else
        snprintf(msg, sizeof msg, "the knot spacing (dt_so3 / dt_r3 ratio) gives a half bandwidth of %d columns over %d knot columns: no elimination "
                 "plan of the solver fits in shared memory at any sequence length (half bandwidths from 112 never fit; use a knot-spacing "
                 "ratio closer to 1)", kd, nk);
      return fail(h, ICC_ERR_UNSUPPORTED, msg);
    }
  }
  DeviceProblem& P = h->P;
  P.nk = nk; P.nb = nb; P.kd = kd; P.ldb = kd + 1;
  P.col_tic = h->col_tic; P.col_g = h->col_g; P.col_ld = h->col_ld; P.col_ai = col_ai; P.col_gi = col_gi; P.col_ci = col_ci; P.col_to = col_to; P.col_pts = col_pts; P.n_points = npts;
  P.bias_active = (ab || gb) ? 1 : 0; P.intr_active = (intr || toff) ? 1 : 0; P.cam_intr_active = cam_intr ? 1 : 0;
  P.ne_off_E = (int64_t)nk * P.ldb; P.ne_off_C = P.ne_off_E + (int64_t)nk * nb; P.ne_off_g = P.ne_off_C + (int64_t)nb * nb;
  P.ne_off_cost = P.ne_off_g + nk + nb; P.ne_size = (P.ne_off_cost + 1 + 3) / 4 * 4;
  if (h->device >= 0) {
    // (staged through the page-locked arena while it has room: asynchronous, ordered before the kernels on the solver's stream)
    CU(upload_staged(h, h->d_so3_col, h->so3_col)); CU(upload_staged(h, h->d_r3_col, h->r3_col)); CU(upload_staged(h, h->d_ba_col, h->ba_col)); CU(upload_staged(h, h->d_bg_col, h->bg_col));
    P.so3_col = h->d_so3_col.p; P.r3_col = h->d_r3_col.p; P.ba_col = h->d_ba_col.p; P.bg_col = h->d_bg_col.p;
    CU(h->d_ne.alloc((size_t)P.ne_size)); P.ne = h->d_ne.p;
    CU(h->d_incr.alloc((size_t)INCR_DOUBLES * std::max(1, P.n_so3 - 1))); P.incr = h->d_incr.p;
    CU(h->d_scale.alloc((size_t)std::max(1, nk + nb))); CU(h->d_delta.alloc((size_t)std::max(1, nk + nb)));
    CU(h->d_ws.alloc(solve_workspace_doubles(P, 0)));
  }
  h->cur_flags = flags;
  return ICC_OK;
}

extern "C" int icc_comm_allreduce_sum(icc_comm* c, double* dev, int64_t n, void* stream);
// Cross-rank sum of a device buffer on the solver's stream: the library's own NCCL communicator, else the caller's hook.  Every rank
// must enter every sum (also with an empty slice), and a failing collective fails the call.
icc_status cross_rank_sum(icc_handle* h, double* dev, int64_t n) {
  if (h->shard_world <= 1) return ICC_OK;
  if (h->comm) return icc_comm_allreduce_sum(h->comm, dev, n, (void*)h->stream) ? fail(h, ICC_ERR_CUDA, std::string("all-reduce failed: ") + icc_comm_last_error()) : ICC_OK;
  if (h->allreduce) { h->allreduce(dev, n, (void*)h->stream, h->allreduce_user); return ICC_OK; }
  return ICC_OK;   // shards evaluated on their own (tests add them up on the host)
}

// the tangent measurements the evaluation kernels take in tangent mode; nullptr selects the pixel residual
const TangentMeas* tangent_meas(const icc_handle* h) { return h->reproj_error == ICC_REPROJ_ERROR_TANGENT ? &h->tan : nullptr; }

// The random-walk prior of the bias splines with its rows placed after the gyroscope rows of the residual vector
BiasPrior prior_at(const icc_handle* h) {
  BiasPrior B = h->prior;
  const int base = h->P.n_res_vis + h->P.n_res_acc + h->P.n_res_gyr;
  B.res_off[0] += base; B.res_off[1] += base;
  return B;
}

// One Jacobian evaluation on the current state: zero the packed normal equations, run the kernels, add the bias prior (when set),
// cross-rank reduce.
icc_status eval_jacobian(icc_handle* h, const DeviceState& S, double* residuals_dev) {
  h->ne_flags = -1;
  CU(cudaMemsetAsync(h->P.ne, 0, (size_t)h->P.ne_size * sizeof(double), h->stream));
  if (launch_eval(h->P, S, true, nullptr, residuals_dev, nullptr, h->stream, h->aux_ok ? &h->aux : nullptr, tangent_meas(h))) return fail(h, ICC_ERR_CUDA, std::string("eval launch: ") + cudaGetErrorString(cudaGetLastError()));
  if (h->P.col_pts >= 0 && h->P.rolling) launch_points_jac(h->P, S, S.pjac, h->P.col_pts, h->sm_count, h->stream, tangent_meas(h));   // board-point columns (POINTS)
  launch_bias_prior(prior_at(h), h->P, S, true, nullptr, residuals_dev, h->stream);
  return cross_rank_sum(h, h->P.ne, h->P.ne_size);
}
icc_status eval_cost(icc_handle* h, const DeviceState& S, double* cost_dev, double* residuals_dev, double* reproj_dev) {
  if (launch_eval(h->P, S, false, cost_dev, residuals_dev, reproj_dev, h->stream, h->aux_ok ? &h->aux : nullptr, tangent_meas(h))) return fail(h, ICC_ERR_CUDA, std::string("eval launch: ") + cudaGetErrorString(cudaGetLastError()));
  launch_bias_prior(prior_at(h), h->P, S, false, cost_dev, residuals_dev, h->stream);
  return cost_dev ? cross_rank_sum(h, cost_dev, 1) : ICC_OK;
}

icc_status mean_reproj(icc_handle* h, double* out) {
  // GetMeanReprojectionError (impl.h:993-1072): RS functor on every view, values only
  if (h->P.n_vwork == 0 && h->shard_world <= 1) { *out = 0.0; return ICC_OK; }
  CU(cudaMemsetAsync(h->d_scal.p, 0, SC_COUNT * sizeof(double), h->stream));
  if (h->P.n_vwork > 0) {
    DeviceProblem P = h->P; P.n_iwork = 0; P.rolling = 1;   // the pixel residual in either mode (no TangentMeas)
    if (launch_eval(P, h->st[h->cur].view(), false, h->d_scal.p + SC_CAND_COST, nullptr, h->d_scal.p + SC_REPROJ_SUM, h->stream)) return fail(h, ICC_ERR_CUDA, "eval launch failed");
  }
  { icc_status r = cross_rank_sum(h, h->d_scal.p + SC_REPROJ_SUM, 2); if (r != ICC_OK) return r; }   // a rank without vision work still enters the sum
  double sc[SC_COUNT];
  CU(cudaMemcpyAsync(sc, h->d_scal.p, sizeof sc, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  if (!(sc[SC_REPROJ_CNT] > 0.0)) { *out = 0.0; return ICC_OK; }
  *out = sc[SC_REPROJ_SUM] / sc[SC_REPROJ_CNT];
  return ICC_OK;
}

// configure() accepted the knot band, so a plan that does not fit is the border's doing; with free bias knots the message names their
// count and spacing, the usual cause (icc_set_bias_splines)
std::string border_too_wide_message(const icc_handle* h) {
  const DeviceProblem& P = h->P;
  char msg[512];
  int len = snprintf(msg, sizeof msg, "the border of %d columns (globals, bias knots, board points) is too wide for the solver's shared-memory plans "
                     "(half bandwidth %d, %d knot columns)", P.nb, P.kd, P.nk);
  const bool ab = !h->ba_col.empty() && h->ba_col[0] >= 0, gb = !h->bg_col.empty() && h->bg_col[0] >= 0;
  if ((ab || gb) && len > 0 && len < (int)sizeof msg)
    snprintf(msg + len, sizeof msg - len, "; %d of them are columns of free bias knots: %d accelerometer knots at %g s spacing, %d gyroscope knots at %g s spacing "
             "(a wider spacing, icc_set_bias_splines, gives fewer)", 3 * ((ab ? P.n_ba : 0) + (gb ? P.n_bg : 0)), ab ? P.n_ba : 0, double(h->dt_ba_ns) / S_TO_NS,
             gb ? P.n_bg : 0, double(h->dt_bg_ns) / S_TO_NS);
  return msg;
}

// Levenberg-Marquardt with Ceres TrustRegionMinimizer semantics (options: impl.h:254-266 + Ceres 2.1 defaults).
icc_status run_lm(icc_handle* h, int max_iters, int flags, bool check_convergence, icc_summary* out) {
  using clk = std::chrono::steady_clock;
  const auto t_start = clk::now();
  PhaseTrace trace(h->stream);
  icc_status rc = configure(h, flags);
  if (rc != ICC_OK) return rc;
  trace.lap("run_lm: configure");
  icc_summary S; memset(&S, 0, sizeof S);
  const DeviceProblem& P = h->P;
  const int n = P.nk + P.nb;
  S.num_residuals = P.n_res_vis + P.n_res_acc + P.n_res_gyr + h->n_res_prior; S.num_tangent = n;
  const int launches0 = kernel_launch_count();
  std::vector<cudaEvent_t> ev;
  auto mark = [&]() { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, h->stream); ev.push_back(e); return (int)ev.size() - 1; };
  std::vector<std::pair<int, int>> jac_spans, lin_spans;
  double sc[SC_COUNT];
  auto jac = [&]() -> icc_status {
    const int a = mark();
    icc_status r = eval_jacobian(h, h->st[h->cur].view(), nullptr);
    if (r != ICC_OK) return r;
    const int b = mark(); jac_spans.push_back({a, b});
    ++S.jacobian_evaluations;
    return ICC_OK;
  };
  // After a Jacobian evaluation: Jacobi scaling (first time) + gradient max-norm, and the cost at x parked next to the other
  // per-iteration scalars, so that ONE device->host read-back (and one stream synchronisation) serves the whole LM iteration.
  auto after_jacobian = [&](bool compute_scale) -> icc_status {
    CU(cudaMemsetAsync(h->d_scal.p + SC_GRAD_MAX, 0, sizeof(double), h->stream));
    launch_compute_scale(P, compute_scale ? h->d_scale.p : nullptr, h->opt.jacobi_scaling, h->d_scal.p, h->stream);
    return ICC_OK;
  };
  auto read_scalars = [&]() -> icc_status {
    CU(cudaMemcpyAsync(sc, h->d_scal.p, sizeof sc, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return ICC_OK;
  };
  if (n == 0) { if (out) *out = S; return ICC_OK; }
  TrOptions to;
  to.function_tolerance = h->opt.function_tolerance; to.parameter_tolerance = h->opt.parameter_tolerance; to.gradient_tolerance = h->opt.gradient_tolerance;
  to.initial_radius = h->opt.initial_trust_region_radius; to.max_radius = h->opt.max_trust_region_radius; to.min_radius = h->opt.min_trust_region_radius;
  to.min_relative_decrease = h->opt.min_relative_decrease; to.min_diagonal = h->opt.min_lm_diagonal; to.max_diagonal = h->opt.max_lm_diagonal;
  to.max_iterations = max_iters; to.max_invalid = h->opt.max_consecutive_invalid_steps; to.check_convergence = check_convergence ? 1 : 0;
  TrustRegion T = tr_start(to);
  while (tr_continue(T)) {
    // The Jacobian / normal equations are (re)built lazily at the top of the iteration that needs them, so that n
    // iterations cost n linear solves + n cost evaluations + one Jacobian evaluation per accepted step (and the first).
    const bool fresh_jacobian = T.jacobian_stale != 0;
    if (fresh_jacobian) {
      rc = jac(); if (rc != ICC_OK) return rc;
      rc = after_jacobian(T.iterations == 0); if (rc != ICC_OK) return rc;
    }
    SolveParams sp; sp.radius = T.radius; sp.min_diag = to.min_diagonal; sp.max_diag = to.max_diagonal; sp.jacobi_scaling = h->opt.jacobi_scaling;
    const int a = mark();
    { const int se = launch_solve(P, h->d_scale.p, sp, h->d_ws.p, h->d_delta.p, h->d_scal.p, h->stream, 0);
      if (se == 1) return fail(h, ICC_ERR_UNSUPPORTED, border_too_wide_message(h));
      if (se) return fail(h, ICC_ERR_CUDA, std::string("solver launch: ") + cudaGetErrorString(cudaGetLastError())); }
    const int b = mark(); lin_spans.push_back({a, b});
    const int cand = 1 - h->cur;
    launch_update(P, h->st[h->cur].view(), h->st[cand].view(), h->d_delta.p, h->max_ba, h->max_bg, h->d_scal.p, h->stream);
    if (P.col_pts >= 0) launch_points_update(P.n_points, P.col_pts, h->st[h->cur].pts.p, h->st[cand].pts.p, h->st[cand].board.p, h->st[cand].pjac.p, h->d_delta.p, h->d_scal.p, h->stream);
    rc = eval_cost(h, h->st[cand].view(), h->d_scal.p + SC_CAND_COST, nullptr, nullptr); if (rc != ICC_OK) return rc;
    rc = read_scalars(); if (rc != ICC_OK) return rc;
    trace.lap("run_lm: iteration");
    if (fresh_jacobian) {
      if (T.iterations == 0 && !std::isfinite(sc[SC_X_COST])) return fail(h, ICC_ERR_NUMERIC, "non-finite initial cost");
      // Ceres tests the gradient right after the Jacobian evaluation; the step computed above is simply discarded
      if (!tr_jacobian(T, sc[SC_X_COST], sc[SC_GRAD_MAX])) break;
    }
    if (tr_step(T, sc[SC_OK] != 0.0, sc[SC_MODEL_CHANGE], std::sqrt(sc[SC_STEP_SQ]), std::sqrt(sc[SC_X_SQ])) && tr_candidate(T, sc[SC_CAND_COST])) {
      h->cur = cand; h->state_dirty_host = true; h->glob_host_current = false;
    }
  }
  S.termination = T.termination; S.iterations = S.cost_evaluations = T.iterations; S.successful_steps = T.successful;
  S.initial_cost = T.initial_cost; S.final_cost = T.cost;
  if (max_iters <= 0) {   // no iteration ran: the costs at x
    rc = jac(); if (rc != ICC_OK) return rc; rc = after_jacobian(true); if (rc != ICC_OK) return rc; rc = read_scalars(); if (rc != ICC_OK) return rc;
    S.initial_cost = S.final_cost = sc[SC_X_COST];
  }
  if (P.col_pts >= 0 && S.successful_steps > 0) {   // both state buffers carry the accepted points again (runs without POINTS never copy them)
    const StateBufs& a = h->st[h->cur]; StateBufs& b = h->st[1 - h->cur];
    CU(cudaMemcpyAsync(b.pts.p, a.pts.p, a.pts.n * sizeof(double4), cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaMemcpyAsync(b.board.p, a.board.p, a.board.n * sizeof(double4), cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaMemcpyAsync(b.pjac.p, a.pjac.p, a.pjac.n * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  }
  CU(cudaStreamSynchronize(h->stream));
  auto span_s = [&](const std::vector<std::pair<int, int>>& v) { double tot = 0; for (auto& p : v) { float ms = 0; cudaEventElapsedTime(&ms, ev[p.first], ev[p.second]); tot += ms; } return tot * 1e-3; };
  S.seconds_jacobian = span_s(jac_spans); S.seconds_linear_solve = span_s(lin_spans);
  for (auto e : ev) cudaEventDestroy(e);
  S.gpu_launches = kernel_launch_count() - launches0;
  S.seconds_total = std::chrono::duration<double>(clk::now() - t_start).count();
  trace.lap("run_lm: epilogue");
  if (out) *out = S;
  return ICC_OK;
}

// ---- the steps of icc_batch_init_spline ------------------------------------------------------------------------------------------------

struct KnotCounts { int so3, r3, ba, bg; };

// T_i_c, IMU intrinsics, line delay (imu_camera_calibrator.cc:30-47), the spline time range and knot counts (imu_camera_calibrator.cc:49-72,
// impl.h:37-51), and the bias splines: InitBiasSplines(bias, bias, 10 s, 10 s, 1.0, 0.1) (imu_camera_calibrator.cc:80-85, impl.h:53-90).
// The SO(3) / R³ knots are only sized (zero) here.
icc_status init_globals_and_knot_counts(icc_handle* h, KnotCounts& n) {
  const icc_init_params& ip = h->ip;
  { const Q4 q = qn(ip.T_i_c_init); h->glob[G_TIC + 0] = q.x; h->glob[G_TIC + 1] = q.y; h->glob[G_TIC + 2] = q.z; h->glob[G_TIC + 3] = q.w; for (int i = 4; i < 7; ++i) h->glob[G_TIC + i] = ip.T_i_c_init[i]; }
  for (int i = 0; i < 6; ++i) h->glob[G_ACC_INTR + i] = ip.acc_intrinsics[i];
  for (int i = 0; i < 9; ++i) h->glob[G_GYR_INTR + i] = ip.gyr_intrinsics[i];
  h->glob[G_LD] = ip.init_line_delay_s;
  for (int i = 0; i < MAX_INTR; ++i) h->glob[G_CAM_INTR + i] = i < h->n_intr ? h->intr[i] : 0.0;
  h->glob[G_TOFF] = 0.0;
  const auto range = std::minmax_element(h->frame_t.begin(), h->frame_t.end());
  h->t0_s = *range.first; h->tend_s = *range.second;
  h->start_ns = (int64_t)(h->t0_s * S_TO_NS);
  h->end_ns = (int64_t)(h->tend_s * S_TO_NS + 0.01 * S_TO_NS + ip.init_line_delay_s);
  h->dt_so3_ns = (int64_t)(ip.dt_so3_s * S_TO_NS); h->dt_r3_ns = (int64_t)(ip.dt_r3_s * S_TO_NS);
  if (h->dt_so3_ns <= 0 || h->dt_r3_ns <= 0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "knot spacing must be positive");
  // the bias spacing of icc_set_bias_splines in place of the reference's constant 10 s; the bias box stays the reference's
  auto bias_dt_ns = [](double dt_s) { return dt_s > 0.0 ? (int64_t)(dt_s * S_TO_NS) : (int64_t)(10 * 1e9); };
  h->dt_ba_ns = bias_dt_ns(h->bias_dt_s_set[0]); h->dt_bg_ns = bias_dt_ns(h->bias_dt_s_set[1]); h->max_ba = 1.0; h->max_bg = 1e-1;
  const int64_t duration = h->end_ns - h->start_ns;
  n = {(int)(duration / h->dt_so3_ns) + SPLINE_N, (int)(duration / h->dt_r3_ns) + SPLINE_N, (int)(duration / h->dt_ba_ns) + BIAS_N, (int)(duration / h->dt_bg_ns) + BIAS_N};
  {   // the prior rows: shard 0 owns them, so that the cross-rank sums count them once
    BiasPrior& B = h->prior; B = BiasPrior{};
    const int nk[2] = {n.ba, n.bg}; const int64_t dt[2] = {h->dt_ba_ns, h->dt_bg_ns};
    int off = 0;
    for (int s = 0; s < 2; ++s) {
      B.on[s] = h->walk_set[s] && h->shard_rank == 0 ? 1 : 0;
      for (int a = 0; a < 3; ++a) B.c[s][a] = B.on[s] ? bias_prior_scale(double(dt[s]) / S_TO_NS, h->walk_q_set[s][a]) : 0.0;
      B.res_off[s] = off;                                       // relative to the end of the gyroscope rows (see prior_at)
      if (B.on[s]) off += 3 * BIAS_PRIOR_NODES * (nk[s] - 2);
    }
    h->n_res_prior = off;
  }
  h->so3.assign(4 * (size_t)n.so3, 0.0); h->r3.assign(3 * (size_t)n.r3, 0.0);
  h->ba.resize(3 * (size_t)n.ba); h->bg.resize(3 * (size_t)n.bg);
  for (int i = 0; i < n.ba; ++i) for (int d = 0; d < 3; ++d) h->ba[3 * i + d] = ip.acc_bias[d];
  for (int i = 0; i < n.bg; ++i) for (int d = 0; d < 3; ++d) h->bg[3 * i + d] = ip.gyr_bias[d];
  return ICC_OK;
}

// The per-view pose priors (raw q_wc, p_wc) in the order the reference walks its views: through a std::map keyed by timestamp (time order,
// a repeated timestamp keeps the LAST view).  Strictly increasing timestamps -- the usual case -- give that order without the tree.
struct ViewTable { std::vector<double> t, q, p; bool increasing = true; };
ViewTable view_table(const icc_handle* h) {
  const int nf = (int)h->frame_t.size();
  ViewTable v;
  for (int i = 1; i < nf && v.increasing; ++i) v.increasing = h->frame_t[i] > h->frame_t[i - 1];
  std::vector<int> order;
  if (v.increasing) { order.resize(nf); for (int i = 0; i < nf; ++i) order[i] = i; }
  else { std::map<double, int> by_time; for (int i = 0; i < nf; ++i) by_time[h->frame_t[i]] = i; for (const auto& kv : by_time) order.push_back(kv.second); }
  v.t.reserve(order.size()); v.q.reserve(4 * order.size()); v.p.reserve(3 * order.size());
  for (const int i : order) { v.t.push_back(h->frame_t[i]); for (int d = 0; d < 4; ++d) v.q.push_back(h->q_wc[4 * i + d]); for (int d = 0; d < 3; ++d) v.p.push_back(h->p_wc[3 * i + d]); }
  return v;
}

Pose T_c_i(const icc_handle* h) { return pose_inv({q4(h->glob[G_TIC + 0], h->glob[G_TIC + 1], h->glob[G_TIC + 2], h->glob[G_TIC + 3]), v3(h->glob[G_TIC + 4], h->glob[G_TIC + 5], h->glob[G_TIC + 6])}); }

// BatchInitSO3R3VisPoses (impl.h:278-339) for the host-only handle: init_knots_kernel's per-knot functions, into the host mirror
void init_knots_on_host(icc_handle* h, const ViewTable& v, const Pose& Tci) {
  const int nv = (int)v.t.size(), nso3 = (int)h->so3.size() / 4, nr3 = (int)h->r3.size() / 3;
  for (int i = 0; i < nso3; ++i) {
    const double4 o = so3_knot(i, h->dt_so3_ns, nv, v.t.data(), v.q.data(), v.p.data(), Tci.q, Tci.t);
    h->so3[4 * i] = o.x; h->so3[4 * i + 1] = o.y; h->so3[4 * i + 2] = o.z; h->so3[4 * i + 3] = o.w;
  }
  for (int j = 0; j < nr3; ++j) {
    const double4 o = r3_knot(j, h->dt_r3_ns, nr3, nv, v.t.data(), v.q.data(), v.p.data(), Tci.q, Tci.t);
    h->r3[3 * j] = o.x; h->r3[3 * j + 1] = o.y; h->r3[3 * j + 2] = o.z;
  }
}

// CalcTimes of every frame (impl.h:541); `accepted` lists the frames both splines accept, in input order
std::vector<FrameHost> frame_times(icc_handle* h, const KnotCounts& n, std::vector<int>& accepted) {
  const int nf = (int)h->frame_t.size();
  std::vector<FrameHost> frames(nf);
  accepted.clear(); h->dropped_frames = 0;
  for (int i = 0; i < nf; ++i) {
    FrameHost& f = frames[i]; f.t_s = h->frame_t[i]; f.c0 = h->corner_off[i]; f.c1 = h->corner_off[i + 1];
    const int64_t t_ns = (int64_t)(f.t_s * S_TO_NS);
    int64_t s1 = 0, s2 = 0;
    const bool ok = calc_times(t_ns, h->start_ns, h->dt_r3_ns, n.r3, SPLINE_N, f.u_r3, s1) && calc_times(t_ns, h->start_ns, h->dt_so3_ns, n.so3, SPLINE_N, f.u_so3, s2);
    f.s_r3 = (int)s1; f.s_so3 = (int)s2;
    if (ok) accepted.push_back(i); else ++h->dropped_frames;
  }
  return frames;
}

// Kept samples [ka, kb) of a sorted stream, used in place: the cells -- maximal runs of samples inside the same knot interval of all four
// splines -- are found by galloping + bisection for the next interval boundary (CalcTimes' st is monotone in t), so the host touches
// O(cells log run) time stamps instead of every sample.  The relative times st = int64((t + offset) 1e9) - start themselves are derived on
// the device from the uploaded stamps (imu_times_kernel), bit for bit.
void cells_by_bisection(icc_handle* h, size_t ka, size_t kb) {
  const double* imu_t = h->imu_t.data(); const double toff = h->ip.time_offset_imu_to_cam_s;
  auto st_of = [&](size_t i) { return (int64_t)((imu_t[i] + toff) * S_TO_NS) - h->start_ns; };
  h->cells.clear(); h->imu_used_t.clear(); h->imu_used_st.clear();
  size_t k = ka;
  while (k < kb) {
    const int64_t st = st_of(k);
    const int64_t a = st / h->dt_r3_ns, b = st / h->dt_so3_ns, c = st / h->dt_ba_ns, d = st / h->dt_bg_ns;
    const int64_t edge = std::min(std::min((a + 1) * h->dt_r3_ns, (b + 1) * h->dt_so3_ns), std::min((c + 1) * h->dt_ba_ns, (d + 1) * h->dt_bg_ns));
    size_t prev = k, probe = k + 1, step = 1;                     // first index in (k, kb) with st >= edge: gallop, then bisect
    while (probe < kb && st_of(probe) < edge) { prev = probe; probe += step; step *= 2; }
    size_t lo = prev + 1, hi = std::min(probe, kb);                // st_of(prev) < edge <= st_of(probe) (or probe is past the end)
    while (lo < hi) { const size_t m = (lo + hi) / 2; if (st_of(m) < edge) lo = m + 1; else hi = m; }
    h->cells.push_back({(int)b, (int)a, (int)c, (int)d, (int)(k - ka), (int)(lo - ka)});
    k = lo;
  }
  h->imu_lazy = true; h->n_imu_used = kb - ka; h->imu_contig = kb > ka; h->imu_src0 = kb > ka ? (int)ka : 0;
}

// Measurement selection of a time-sorted stream (the usual case; known from set_imu).  CalcTimes' validity tests are monotone in time, so
// the kept samples are ONE index range [ia, ib) of imu_t, found by bisection.  The shard rule -- unit `mine` iff the scalar residuals of all
// units before it in the time-merged order (frames before IMU samples on ties) fall in [lo, hi) -- is then evaluated on counts: frames are
// break points found by bisection, and only the shard's own samples are walked, by cells_by_bisection.  O(frames log samples + cells log
// run) instead of O(samples) per rank; same decisions as select_general (tests/test_capi_boundary.py, test_sharding_gloo.py).  One shard
// keeps every accepted frame (the rule on counts would drop a corner-less frame after the last unit with residuals).  Declines (false) for
// an unsorted stream, a stream without kept samples, and frames out of time order when there are several shards.
bool select_sorted(icc_handle* h, const KnotCounts& n, const std::vector<FrameHost>& frames, const std::vector<int>& accepted, bool frames_increasing,
                   std::vector<int>& frame_sel) {
  if (!h->imu_sorted || (h->shard_world > 1 && !frames_increasing)) return false;
  const size_t n_in = h->imu_t.size();
  const double* imu_t = h->imu_t.data(); const double toff = h->ip.time_offset_imu_to_cam_s, t0 = h->t0_s, tend = h->tend_s;
  auto bisect = [](size_t a, size_t b, auto pred) { while (a < b) { const size_t m = (a + b) / 2; if (pred(m)) a = m + 1; else b = m; } return a; };   // first index where pred is false
  auto fits = [&](size_t i) {   // upper-side validity of CalcTimes for all four splines (monotone: true, then false)
    const double t = imu_t[i] + toff;
    if (t >= tend) return false;
    const int64_t st = (int64_t)(t * S_TO_NS) - h->start_ns;
    return size_t(st / h->dt_r3_ns + SPLINE_N) <= (size_t)n.r3 && size_t(st / h->dt_so3_ns + SPLINE_N) <= (size_t)n.so3 && size_t(st / h->dt_ba_ns + BIAS_N) <= (size_t)n.ba && size_t(st / h->dt_bg_ns + BIAS_N) <= (size_t)n.bg;
  };
  const size_t ia = bisect(0, n_in, [&](size_t i) { const double t = imu_t[i] + toff; return t < t0 || (int64_t)(t * S_TO_NS) - h->start_ns < 0; });
  const size_t ib = bisect(ia, n_in, fits);
  if (ib <= ia) return false;
  const size_t in_window = bisect(ia, n_in, [&](size_t i) { return imu_t[i] + toff < tend; }) - ia;
  h->dropped_imu = (int)(in_window - (ib - ia));
  size_t ka = ia, kb = ib;                  // this shard's samples
  if (h->shard_world == 1) frame_sel = accepted;
  else {
    long total = 6 * (long)(ib - ia);
    for (int j : accepted) total += 2 * (frames[j].c1 - frames[j].c0);
    const long lo = total * h->shard_rank / h->shard_world, hi = total * (h->shard_rank + 1) / h->shard_world;
    auto ceil_div6 = [](long v) { return v <= 0 ? 0L : (v + 5) / 6; };
    ka = ib; kb = ia;
    size_t prev_p = ia;
    long Rf = 0;                            // residuals of the accepted frames seen so far
    auto take_imu = [&](size_t a, size_t b) {   // samples [a, b) lie between two frames: run_before(i) = Rf + 6 (i - ia)
      const size_t first = std::max(a, ia + (size_t)ceil_div6(lo - Rf)), last = std::min(b, ia + (size_t)ceil_div6(hi - Rf));
      if (first < last) { ka = std::min(ka, first); kb = std::max(kb, last); }
    };
    for (int j : accepted) {
      const double tf = frames[j].t_s;
      const size_t p = bisect(prev_p, ib, [&](size_t i) { return imu_t[i] + toff < tf; });   // samples strictly before the frame
      take_imu(prev_p, p);
      const long run = Rf + 6 * (long)(p - ia);
      if (run >= lo && run < hi) frame_sel.push_back(j);
      Rf += 2 * (frames[j].c1 - frames[j].c0);
      prev_p = p;
    }
    take_imu(prev_p, ib);
    if (ka > kb) ka = kb = ia;
  }
  cells_by_bisection(h, ka, kb);
  return true;
}

// CalcTimes' segment index s = st / dt of a time-sorted stream only ever steps forward: track it with comparisons and fall back to the
// division when a sample is not where the previous one left off (unsorted input); the results are identical
struct SegTrack { int64_t dt, s = 0, lo = 0, hi = -1;   // [lo, hi) = time range of segment s; hi < lo until the first sample
  int64_t seg(int64_t st) {
    if (st >= lo && st < hi) return s;
    if (hi > lo && st >= hi && st < hi + 63 * dt) { do { ++s; lo = hi; hi += dt; } while (st >= hi); return s; }
    s = st / dt; lo = s * dt; hi = lo + dt; return s;
  } };

// Measurement selection of any stream: one pass collects the kept samples, frames and samples are merged in time order and cut by the
// shard rule, and the shard's samples are copied (their readings gathered unless they are one contiguous run of the input).
icc_status select_general(icc_handle* h, const KnotCounts& n, const std::vector<FrameHost>& frames, const std::vector<int>& accepted, std::vector<int>& frame_sel) {
  struct ImuHost { double t_s; int64_t st; int s_so3, s_r3, s_ba, s_bg; int src; };
  const size_t n_in = h->imu_t.size();
  std::vector<ImuHost> kept; kept.reserve(n_in);
  {
    SegTrack tr_r3{h->dt_r3_ns}, tr_so3{h->dt_so3_ns}, tr_ba{h->dt_ba_ns}, tr_bg{h->dt_bg_ns};
    h->dropped_imu = 0;
    const double* imu_t = h->imu_t.data(); const double toff = h->ip.time_offset_imu_to_cam_s, t0 = h->t0_s, tend = h->tend_s;
    for (size_t i = 0; i < n_in; ++i) {
      const double t = imu_t[i] + toff;
      if (t < t0 || t >= tend) continue;
      const int64_t t_ns = (int64_t)(t * S_TO_NS), st = t_ns - h->start_ns;
      bool ok = st >= 0;
      int64_t a = 0, b = 0, c = 0, d = 0;
      if (ok) { a = tr_r3.seg(st); b = tr_so3.seg(st); c = tr_ba.seg(st); d = tr_bg.seg(st);
                ok = size_t(a + SPLINE_N) <= (size_t)n.r3 && size_t(b + SPLINE_N) <= (size_t)n.so3 && size_t(c + BIAS_N) <= (size_t)n.ba && size_t(d + BIAS_N) <= (size_t)n.bg; }
      if (!ok) { ++h->dropped_imu; continue; }
      kept.push_back({t, st, (int)b, (int)a, (int)c, (int)d, (int)i});
    }
  }
  struct Unit { double t; int kind, idx, nres; };
  std::vector<Unit> units; units.reserve(accepted.size() + kept.size());
  for (int i : accepted) units.push_back({frames[i].t_s, 0, i, 2 * (frames[i].c1 - frames[i].c0)});
  const size_t nfu = units.size();
  for (size_t i = 0; i < kept.size(); ++i) units.push_back({kept[i].t_s, 1, (int)i, 6});
  {   // time order with frames before IMU samples on ties (== stable sort of [frames..., imu...]); both streams are normally
      // already sorted, so merge in O(n) and only fall back to sorting when they are not
    auto lt = [](const Unit& x, const Unit& y) { return x.t < y.t; };
    if (!std::is_sorted(units.begin(), units.begin() + nfu, lt)) std::stable_sort(units.begin(), units.begin() + nfu, lt);
    if (!std::is_sorted(units.begin() + nfu, units.end(), lt)) std::stable_sort(units.begin() + nfu, units.end(), lt);
    std::vector<Unit> merged(units.size());
    std::merge(units.begin(), units.begin() + nfu, units.begin() + nfu, units.end(), merged.begin(), lt);
    units.swap(merged);
  }
  long total = 0; for (const auto& u : units) total += u.nres;
  const long lo = total * h->shard_rank / h->shard_world, hi = total * (h->shard_rank + 1) / h->shard_world;
  long run = 0;
  std::vector<int> imu_sel;
  frame_sel.clear();
  for (const auto& u : units) { const bool mine = run >= lo && run < hi; run += u.nres; if (!mine) continue; (u.kind == 0 ? frame_sel : imu_sel).push_back(u.idx); }
  std::sort(frame_sel.begin(), frame_sel.end());
  h->imu_lazy = false; h->n_imu_used = imu_sel.size();
  h->imu_contig = !imu_sel.empty();
  for (size_t k = 1; k < imu_sel.size() && h->imu_contig; ++k) h->imu_contig = kept[imu_sel[k]].src == kept[imu_sel[k - 1]].src + 1;
  h->imu_src0 = imu_sel.empty() ? 0 : kept[imu_sel.front()].src;
  h->imu_used_t.resize(imu_sel.size()); h->imu_used_st.resize(imu_sel.size(), h->device >= 0);
  if (!h->imu_contig) { icc_status es = ensure_host_imu(h); if (es != ICC_OK) return es; }
  if (!h->imu_contig) { h->imu_used_acc.resize(3 * imu_sel.size()); h->imu_used_gyr.resize(3 * imu_sel.size()); }
  h->cells.clear();
  for (size_t k = 0; k < imu_sel.size(); ++k) {
    const ImuHost& m = kept[imu_sel[k]];
    const int idx = (int)k;
    h->imu_used_t[k] = m.t_s; h->imu_used_st[k] = m.st;
    if (!h->imu_contig) { memcpy(&h->imu_used_acc[3 * k], &h->imu_acc[3 * (size_t)m.src], 3 * sizeof(double)); memcpy(&h->imu_used_gyr[3 * k], &h->imu_gyr[3 * (size_t)m.src], 3 * sizeof(double)); }
    if (h->cells.empty() || h->cells.back().s_so3 != m.s_so3 || h->cells.back().s_r3 != m.s_r3 || h->cells.back().s_ba != m.s_ba || h->cells.back().s_bg != m.s_bg)
      h->cells.push_back({m.s_so3, m.s_r3, m.s_ba, m.s_bg, idx, idx});
    h->cells.back().i_end = idx + 1;
  }
  return ICC_OK;
}

// The corners of the selected frames: used in place when the frames are one contiguous run (the usual case: all frames, or one contiguous
// shard), else gathered on the host
icc_status gather_corners(icc_handle* h, const std::vector<FrameHost>& frames, const std::vector<int>& frame_sel) {
  h->frames.clear(); h->used_uv.clear(); h->used_pid.clear();
  h->frames.reserve(frame_sel.size()); h->corners_rejected = false; h->n_corners_assembled = h->n_corners_in;
  h->frame_in.clear(); for (int fi : frame_sel) h->frame_in.push_back({frames[fi].c0, frames[fi].c1});
  bool consecutive = !frame_sel.empty();
  for (size_t k = 1; k < frame_sel.size() && consecutive; ++k) consecutive = frame_sel[k] == frame_sel[k - 1] + 1;
  h->used_contig = consecutive; h->used_c0 = 0; h->used_n = 0;
  if (consecutive) {
    const int cb = frames[frame_sel.front()].c0, ce = frames[frame_sel.back()].c1;
    h->used_c0 = cb; h->used_n = ce - cb;
    for (int fi : frame_sel) { FrameHost f = frames[fi]; f.c0 -= cb; f.c1 -= cb; h->frames.push_back(f); }
  } else {
    { icc_status es = ensure_host_corners(h); if (es != ICC_OK) return es; }
    for (int fi : frame_sel) {
      FrameHost f = frames[fi];
      const int c0 = (int)h->used_pid.size();
      for (int c = f.c0; c < f.c1; ++c) { h->used_pid.push_back(h->point_ids[c]); h->used_uv.push_back(h->uv[2 * c]); h->used_uv.push_back(h->uv[2 * c + 1]); }
      f.c0 = c0; f.c1 = (int)h->used_pid.size();
      h->frames.push_back(f);
    }
    h->used_n = (int)h->used_pid.size();
  }
  return ICC_OK;
}

// Gravity initialisation (imu_camera_calibrator.cc:130-161) incl. the integer-second truncation of the accelerometer time: the reference
// visits the sorted camera timestamps; a repeated one names the same view (the map's) again and finds nothing new, so each view is
// visited once, in time order
icc_status init_gravity(icc_handle* h, const ViewTable& v, const Pose& Tci) {
  bool ginit = false; double g0[3] = {0.0, 0.0, 9.81};   // GRAVITY_MAGN (spline_trajectory_estimator.h:29) when never initialised
  for (size_t k = 0; k < v.t.size() && !ginit; ++k) {
    const Pose Tai = view_T_w_i(v.q.data(), v.p.data(), (int)k, Tci.q, Tci.t);
    for (size_t i = 0; i < h->imu_t.size(); ++i) {
      const int64_t accl_t = (int64_t)h->imu_t[i];
      if (std::fabs(double(accl_t) - v.t[k]) < 1. / 30.) {
        double a3[3];
        if (h->imu_dev && h->imu_acc.size() != 3 * h->n_imu_in) { CU(cudaMemcpy(a3, h->d_acc_all.p + 3 * i, sizeof a3, cudaMemcpyDeviceToHost)); }   // one reading
        else { a3[0] = h->imu_acc[3 * i]; a3[1] = h->imu_acc[3 * i + 1]; a3[2] = h->imu_acc[3 * i + 2]; }
        const V3 g = qrot(Tai.q, v3(a3[0], a3[1], a3[2])); g0[0] = g.x; g0[1] = g.y; g0[2] = g.z; ginit = true; break; }
    }
  }
  for (int d = 0; d < 3; ++d) h->glob[G_GRAV + d] = g0[d];
  return ICC_OK;
}

// Schedule of the persistent evaluation kernel (icc_eval_tmem.cu).  Both streams -- the corners of the non-empty frames and the samples of
// the knot-interval cells, units padded to a multiple of 4 = one m8n8k4 k-step -- are walked with the kernel's own chunk rule (a chunk = up
// to 32 stream positions from at most two consecutive units) and cut into even per-warp runs: h->vitems / h->iitems and the stream counts
// of h->P.  Returns the unit tables the kernel reads.
struct EvalStreams { std::vector<VisFrame> vf; std::vector<ImuCellP> ic; };
EvalStreams eval_schedule(icc_handle* h) {
  DeviceProblem& P = h->P;
  struct Walk { std::vector<int> pos, unit; int total = 0; };
  auto walk = [](const std::vector<int>& poff, int n_units) { Walk w; w.total = poff[n_units];
    for (int pos = 0, u = 0; pos < w.total;) {
      while (poff[u + 1] <= pos) ++u;
      w.pos.push_back(pos); w.unit.push_back(u);
      const int nA = std::min(32, poff[u + 1] - pos);
      int n = nA;
      if (nA < 32 && u + 1 < n_units) n += std::min(32 - nA, poff[u + 2] - poff[u + 1]);
      pos += n;
    }
    return w; };
  EvalStreams es;
  std::vector<VisFrame>& vf = es.vf; vf.reserve(h->frames.size() + 2);
  std::vector<int> vpoff;
  int poff = 0;
  if (P.rolling) for (const auto& f : h->frames) {
    const int cn = f.c1 - f.c0;
    if (cn <= 0) continue;
    vf.push_back({poff, f.c0, cn, f.s_so3, f.s_r3, 0, f.u_so3, f.u_r3}); vpoff.push_back(poff);
    poff += (cn + 3) / 4 * 4;
  }
  const int nvf = (int)vf.size();
  vf.push_back({poff, 0, 0, 0, 0, 0, 0.0, 0.0}); vf.push_back({poff, 0, 0, 0, 0, 0, 0.0, 0.0});   // sentinels [n], [n+1]
  vpoff.push_back(poff); vpoff.push_back(poff);
  std::vector<ImuCellP>& ic = es.ic; ic.reserve(h->cells.size() + 2);
  std::vector<int> ipoff;
  poff = 0;
  for (const auto& c : h->cells) {
    const int n = c.i_end - c.i_begin;
    if (n <= 0) continue;
    ic.push_back({poff, c.i_begin, n, c.s_so3, c.s_r3, c.s_ba, c.s_bg, 0}); ipoff.push_back(poff);
    poff += (n + 3) / 4 * 4;
  }
  const int nic = (int)ic.size();
  ic.push_back({poff, 0, 0, 0, 0, 0, 0, 0}); ic.push_back({poff, 0, 0, 0, 0, 0, 0, 0});
  ipoff.push_back(poff); ipoff.push_back(poff);
  const Walk wv = walk(vpoff, nvf), wi = walk(ipoff, nic);
  // at most one run per warp of the item type's persistent launch (one CTA per SM)
  int cap = INT_MAX;   // ICC_TMEM_RUNS=n caps the runs at n (tests: every warp then owns several chunks and carries its tile state between them)
  if (const char* e = getenv("ICC_TMEM_RUNS")) { const int n = atoi(e); if (n > 0) cap = n; }
  auto split = [h, cap](const Walk& w, bool imu) {      // even runs, one per warp
    const int W = std::min(h->sm_count * eval_tmem_warps(imu), cap);
    const int nc = (int)w.pos.size(), n_items = std::min(W, nc);
    std::vector<VisItem> items((size_t)n_items);
    for (int k = 0; k < n_items; ++k) {
      const int a = (int)((int64_t)nc * k / n_items), b = (int)((int64_t)nc * (k + 1) / n_items);
      items[(size_t)k] = {w.unit[a], w.pos[a], b < nc ? w.pos[b] : w.total, 0};
    }
    return items; };
  h->vitems = split(wv, false); h->iitems = split(wi, true);
  P.n_vchunks = (int)wv.pos.size(); P.n_ichunks = (int)wi.pos.size();
  P.n_vframes = nvf; P.n_vitems = (int)h->vitems.size(); P.n_icells = nic; P.n_iitems = (int)h->iitems.size();
  return es;
}

// work lists: one warp per item; items sized so that the grid fills the GPU but every item amortises its tile flush
int work_items_target(const icc_handle* h) { return h->sm_count * 8; }
int round32(long v) { return (int)((v + 31) / 32 * 32); }
// the one-warp vision kernels' items: runs of at most per_v corners of one frame (after batch_init and after a corner rejection)
icc_status upload_vision_work(icc_handle* h) {
  DeviceProblem& P = h->P;
  const int per_v = std::max(32, round32(P.n_corners / std::max(1, work_items_target(h))));
  std::vector<VisionWork> vw;
  for (int fi = 0; fi < P.n_frames; ++fi) for (int c = h->frames[fi].c0; c < h->frames[fi].c1; c += per_v) vw.push_back({fi, c, std::min(c + per_v, h->frames[fi].c1), 0});
  CU(upload_staged(h, h->d_vwork, vw)); P.vwork = h->d_vwork.p; P.n_vwork = (int)vw.size();
  return ICC_OK;
}
// the persistent kernel's unit tables and per-warp runs (eval_schedule)
icc_status upload_schedule(icc_handle* h, const EvalStreams& es) {
  DeviceProblem& P = h->P;
  CU(upload_staged(h, h->d_vframes, es.vf)); P.vframes = h->d_vframes.p;
  CU(upload_staged(h, h->d_vitems, h->vitems)); P.vitems = h->d_vitems.p;
  CU(upload_staged(h, h->d_icells, es.ic)); P.icells = h->d_icells.p;
  CU(upload_staged(h, h->d_iitems, h->iitems)); P.iitems = h->d_iitems.p;
  return ICC_OK;
}

// Device upload: the problem arrays and work lists, both state copies, and the knots by init_knots_kernel from the view table.  The small
// arrays are staged through the pinned arena: its size below must cover everything staged through it until the next batch_init (each
// array takes a multiple of 256 bytes), else upload_staged falls back to blocking copies.  A corner rejection restarts the arena once the
// stream has drained and stages only the vision work list and the schedule again, both within what this budget gives them.
icc_status upload_problem(icc_handle* h, const ViewTable& v, const Pose& Tci, const EvalStreams& es, PhaseTrace& trace) {
  DeviceProblem& P = h->P;
  const size_t nf = h->frame_t.size();
  CU(cudaSetDevice(h->device));
  CU(cudaStreamSynchronize(h->stream));   // nothing may still read the staging arena of an earlier call
  trace.lap("batch_init: gravity init");
  h->arena.reset((size_t)(1 << 17) + 64 * nf + 48 * (nf + 4) + 16 * (size_t)(h->sm_count * 16 + 16) + 48 * (nf + h->used_n / 32 + 64) + (96 + 40) * (h->cells.size() + (size_t)P.n_imu / 32 + 64)
                 + 8 * 8 * (nf + 8) + 2 * 40 * (size_t)(P.n_so3 + P.n_r3 + P.n_ba + P.n_bg + 16) + 3 * (32 * (h->points.size() / 4 + 8) + 256) + 3 * (4 * (size_t)(P.n_so3 + P.n_r3 + P.n_ba + P.n_bg) + 1024), true);
  trace.lap("batch_init: pinned arena");
  {
    std::vector<double4> board(h->points.size() / 4);
    // hnormalized(T^-1 X_h) of the functor (residuals.h:357-362) == T^-1 (X / w): the division is done once here
    for (size_t i = 0; i < board.size(); ++i) { const double iw = 1.0 / h->points[4 * i + 3]; board[i] = make_double4(h->points[4 * i] * iw, h->points[4 * i + 1] * iw, h->points[4 * i + 2] * iw, 1.0); }
    CU(upload_staged(h, h->d_board, board)); P.board = h->d_board.p;   // (the evaluation kernels read the copy that belongs to the state: DeviceState::board)
    std::vector<int> off, s1, s2; std::vector<double> u1, u2;
    for (const auto& f : h->frames) { off.push_back(f.c0); s1.push_back(f.s_so3); s2.push_back(f.s_r3); u1.push_back(f.u_so3); u2.push_back(f.u_r3); }
    off.push_back(P.n_corners);
    CU(upload_staged(h, h->d_f_off, off)); CU(upload_staged(h, h->d_f_s_so3, s1)); CU(upload_staged(h, h->d_f_s_r3, s2)); CU(upload_staged(h, h->d_f_u_so3, u1)); CU(upload_staged(h, h->d_f_u_r3, u2));
    P.f_off = h->d_f_off.p; P.f_s_so3 = h->d_f_s_so3.p; P.f_s_r3 = h->d_f_s_r3.p; P.f_u_so3 = h->d_f_u_so3.p; P.f_u_r3 = h->d_f_u_r3.p;
    const bool corners_in_place = h->frames_dev && h->used_contig;   // already on the device (set_frames): used where they lie
    if (corners_in_place) { P.uv = h->d_uv_all.p + h->used_c0; P.pid = h->d_pid_all.p + h->used_c0; }
    else { CU(h->d_uv.alloc(P.n_corners)); CU(h->d_pid.alloc(P.n_corners)); P.uv = h->d_uv.p; P.pid = h->d_pid.p; }   // (u, v) pairs are already laid out as double2
    if (P.n_corners > 0 && !corners_in_place) {
      const double* uv_src = h->used_contig ? h->uv.data() + 2 * (size_t)h->used_c0 : h->used_uv.data();
      const int* pid_src = h->used_contig ? h->point_ids.data() + h->used_c0 : h->used_pid.data();
      // page-locked sources (HostBuf): the DMA transfers run behind the rest of this function; kernels follow on the same stream
      CU(cudaMemcpyAsync(h->d_uv.p, uv_src, (size_t)P.n_corners * sizeof(double2), cudaMemcpyHostToDevice, h->stream));
      CU(cudaMemcpyAsync(h->d_pid.p, pid_src, (size_t)P.n_corners * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    }
    if (h->reproj_error == ICC_REPROJ_ERROR_TANGENT) {   // bearings of this shard's corners under the intrinsics of the start, and the pixel scale of the tangent residuals
      CU(h->d_bear.alloc(P.n_corners)); CU(h->d_bear_ok.alloc(P.n_corners));
      launch_bearings(h->model, h->intr, P.n_corners, P.uv, h->d_bear.p, h->d_bear_ok.p, h->stream);
      h->tan = TangentMeas{h->d_bear.p, h->d_bear_ok.p, tangent_scale(h->model, h->intr, P.dispatch_fov != 0)};
    }
    { icc_status r = upload_vision_work(h); if (r != ICC_OK) return r; }
    const int per_i = std::max(32, round32(P.n_imu / std::max(1, work_items_target(h))));
    std::vector<ImuCell> iw;
    for (const auto& c : h->cells) for (int i = c.i_begin; i < c.i_end; i += per_i) { ImuCell s = c; s.i_begin = i; s.i_end = std::min(i + per_i, c.i_end); iw.push_back(s); }
    CU(upload_staged(h, h->d_iwork, iw)); P.iwork = h->d_iwork.p; P.n_iwork = (int)iw.size();
    CU(upload_staged(h, h->d_cells, h->cells)); P.cells = h->d_cells.p;
    { icc_status r = upload_schedule(h, es); if (r != ICC_OK) return r; }
    CU(h->d_imu_t.alloc(h->n_imu_used));
    if (h->imu_lazy && h->n_imu_used) {   // sorted stream: the raw stamps go up, the relative integer times are derived there
      CU(h->d_imu_traw.alloc(h->n_imu_used));
      CU(cudaMemcpyAsync(h->d_imu_traw.p, h->imu_t.data() + h->imu_src0, h->n_imu_used * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      launch_imu_times((int)h->n_imu_used, h->d_imu_traw.p, h->ip.time_offset_imu_to_cam_s, h->start_ns, h->d_imu_t.p, h->stream);
    } else if (h->n_imu_used) CU(cudaMemcpyAsync(h->d_imu_t.p, h->imu_used_st.data(), h->n_imu_used * sizeof(int64_t), cudaMemcpyHostToDevice, h->stream));
    const bool imu_in_place = h->imu_dev && h->imu_contig;   // already on the device (set_imu): used where they lie
    if (imu_in_place) { P.imu_acc = h->d_acc_all.p + 3 * (size_t)h->imu_src0; P.imu_gyr = h->d_gyr_all.p + 3 * (size_t)h->imu_src0; }
    else { CU(h->d_imu_acc.alloc(3 * (size_t)P.n_imu)); CU(h->d_imu_gyr.alloc(3 * (size_t)P.n_imu)); P.imu_acc = h->d_imu_acc.p; P.imu_gyr = h->d_imu_gyr.p; }
    if (P.n_imu > 0 && !imu_in_place) {
      const double* a_src = h->imu_contig ? h->imu_acc.data() + 3 * (size_t)h->imu_src0 : h->imu_used_acc.data();
      const double* g_src = h->imu_contig ? h->imu_gyr.data() + 3 * (size_t)h->imu_src0 : h->imu_used_gyr.data();
      CU(cudaMemcpyAsync(h->d_imu_acc.p, a_src, 3 * (size_t)P.n_imu * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CU(cudaMemcpyAsync(h->d_imu_gyr.p, g_src, 3 * (size_t)P.n_imu * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    }
    P.imu_t_ns = h->d_imu_t.p;
  }
  trace.lap("batch_init: problem upload");
  icc_status s = upload_state(h, 0, true); if (s != ICC_OK) return s;
  s = upload_state(h, 1, true); if (s != ICC_OK) return s;
  trace.lap("batch_init: state upload");
  {   // knots: BatchInitSO3R3VisPoses on the device, written into both state copies (the zero knots uploaded above only sized them)
    CU(upload_staged(h, h->d_view_t, v.t)); CU(upload_staged(h, h->d_view_q, v.q)); CU(upload_staged(h, h->d_view_p, v.p));
    const double Tci7[7] = {Tci.q.x, Tci.q.y, Tci.q.z, Tci.q.w, Tci.t.x, Tci.t.y, Tci.t.z};
    launch_init_knots((int)v.t.size(), h->d_view_t.p, h->d_view_q.p, h->d_view_p.p, Tci7, P.n_so3, h->dt_so3_ns, P.n_r3, h->dt_r3_ns,
                      h->st[0].so3.p, h->st[1].so3.p, h->st[0].r3.p, h->st[1].r3.p, h->stream);
    h->knots_dirty_host = true;     // the device holds the knots; the host mirror is refreshed on demand (getters / setters)
  }
  trace.lap("batch_init: knot init");
  return ICC_OK;
}


// ---- outlier corners (icc_get_corner_errors / icc_reject_outlier_corners) ------------------------------------------------------------------
template <class T> void swap_dev(DevBuf<T>& a, DevBuf<T>& b) { std::swap(a.p, b.p); std::swap(a.n, b.n); std::swap(a.cap_bytes, b.cap_bytes); }

// Residual pair of every corner at the current state (the cost-only vision kernel, rolling-shutter timing in either shutter mode, the
// residual of the solve: tangent or pixel), then e = |pair| per corner into d_cerr and {sum e^2, count, failed} into d_osum[0..2]
icc_status corner_error_pass(icc_handle* h) {
  const DeviceProblem& P = h->P;
  const int n = P.n_corners;
  CU(h->d_osum.alloc(4)); CU(cudaMemsetAsync(h->d_osum.p, 0, 4 * sizeof(double), h->stream));
  CU(h->d_cres.alloc(2 * (size_t)n)); CU(h->d_cerr.alloc((size_t)n));
  if (n > 0 && P.n_vwork > 0) {
    DeviceProblem Q = P; Q.n_iwork = 0; Q.rolling = 1;
    if (launch_eval(Q, h->st[h->cur].view(), false, nullptr, h->d_cres.p, nullptr, h->stream, nullptr, tangent_meas(h))) return fail(h, ICC_ERR_CUDA, std::string("eval launch: ") + cudaGetErrorString(cudaGetLastError()));
    launch_corner_errors(n, h->d_cres.p, h->d_cerr.p, h->d_osum.p, h->stream);
  }
  return ICC_OK;
}

icc_status reject_outliers(icc_handle* h, double k_sigma, double min_px, icc_outlier_summary* out) {
  DeviceProblem& P = h->P;
  const int n = P.n_corners, nf = P.n_frames;
  const bool tangent = h->reproj_error == ICC_REPROJ_ERROR_TANGENT;
  { icc_status r = corner_error_pass(h); if (r != ICC_OK) return r; }
  double sums[4] = {0.0, 0.0, 0.0, double(n)};
  CU(cudaMemcpyAsync(h->d_osum.p + 3, sums + 3, sizeof(double), cudaMemcpyHostToDevice, h->stream));
  { icc_status r = cross_rank_sum(h, h->d_osum.p, 4); if (r != ICC_OK) return r; }   // every rank enters, with or without corners
  CU(cudaMemcpyAsync(sums, h->d_osum.p, sizeof sums, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  const double rms = sums[1] > 0.0 ? std::sqrt(sums[0] / sums[1]) : 0.0, thr = std::max(min_px, k_sigma * rms);
  int n_new = n, emptied = 0;
  if (n > 0) {
    CU(h->d_ckept.alloc((size_t)nf)); CU(h->d_foff_new.alloc((size_t)nf + 1));
    CU(h->d_uv_new.alloc((size_t)n)); CU(h->d_pid_new.alloc((size_t)n)); CU(h->d_csrc_new.alloc((size_t)n));
    if (tangent) { CU(h->d_bear_new.alloc((size_t)n)); CU(h->d_bear_ok_new.alloc((size_t)n)); }
    if (!h->corners_rejected) {   // the corners still lie as assembled: the input index follows from each frame's first input corner
      std::vector<int> in_off(nf); for (int k = 0; k < nf; ++k) in_off[k] = h->frame_in[k].first;
      CU(h->d_in_off.upload(in_off));
    }
    CornerCompaction C{nf, thr, P.f_off, h->d_cres.p, h->d_cerr.p, P.uv, P.pid, tangent ? h->tan.bear : nullptr, tangent ? h->tan.ok : nullptr,
                       h->corners_rejected ? h->d_csrc.p : nullptr, h->d_in_off.p, h->d_ckept.p, h->d_foff_new.p, h->d_uv_new.p, h->d_pid_new.p,
                       tangent ? h->d_bear_new.p : nullptr, tangent ? h->d_bear_ok_new.p : nullptr, h->d_csrc_new.p};
    launch_compact_corners(C, h->stream);
    std::vector<int> kept((size_t)nf);   // the only per-frame data that comes back
    CU(cudaMemcpyAsync(kept.data(), h->d_ckept.p, (size_t)nf * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->arena.reset(0, true);   // the stream has drained: every staged copy is done, so the vision tables below are staged from the arena's start
    // the compacted arrays become the problem's own (the inputs of icc_set_frames, d_uv_all included, are never written)
    swap_dev(h->d_uv, h->d_uv_new); swap_dev(h->d_pid, h->d_pid_new); swap_dev(h->d_csrc, h->d_csrc_new); swap_dev(h->d_f_off, h->d_foff_new);
    if (tangent) { swap_dev(h->d_bear, h->d_bear_new); swap_dev(h->d_bear_ok, h->d_bear_ok_new); h->tan.bear = h->d_bear.p; h->tan.ok = h->d_bear_ok.p; }
    h->corners_rejected = true;
    int c = 0;
    for (int k = 0; k < nf; ++k) {
      FrameHost& f = h->frames[k];
      if (f.c1 > f.c0 && kept[k] == 0) ++emptied;
      f.c0 = c; c += kept[k]; f.c1 = c;
    }
    n_new = c;
    P.uv = h->d_uv.p; P.pid = h->d_pid.p; P.f_off = h->d_f_off.p;
    P.n_corners = n_new; P.n_res_vis = P.rolling ? 2 * n_new : 0;
    { icc_status r = upload_vision_work(h); if (r != ICC_OK) return r; }
    const EvalStreams es = eval_schedule(h);
    { icc_status r = upload_schedule(h, es); if (r != ICC_OK) return r; }
    h->ne_flags = -1;
  }
  double moved[2] = {double(n - n_new), double(emptied)};
  if (h->shard_world > 1) {
    CU(cudaMemcpyAsync(h->d_osum.p, moved, sizeof moved, cudaMemcpyHostToDevice, h->stream));
    { icc_status r = cross_rank_sum(h, h->d_osum.p, 2); if (r != ICC_OK) return r; }
    CU(cudaMemcpyAsync(moved, h->d_osum.p, sizeof moved, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
  }
  if (out) {
    out->n_corners = (int64_t)llround(sums[3]); out->n_rejected = (int64_t)llround(moved[0]); out->n_failed = (int64_t)llround(sums[2]);
    out->n_frames_emptied = (int32_t)llround(moved[1]); out->rms_px = rms; out->threshold_px = thr;
  }
  return ICC_OK;
}

}  // namespace

// =================================================================================================================
extern "C" {

const char* icc_version(void) { return "icc_b200 0.1 (sm_90a, fp64)"; }

void icc_default_solver_options(icc_solver_options* o) {
  o->function_tolerance = 1e-4; o->parameter_tolerance = 1e-7; o->gradient_tolerance = 1e-10;
  o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32; o->jacobi_scaling = 1; o->max_consecutive_invalid_steps = 5;
}

// device_ordinal >= 0 binds a GPU (required for every compute entry point).  device_ordinal == -1 creates a host-only
// handle whose sole use is inspecting the problem ASSEMBLY (knot initialisation, counts) without a GPU; it cannot compute.
icc_status icc_create(icc_handle** out, int device_ordinal) {
  if (!out) return ICC_ERR_INVALID_ARGUMENT;
  icc_handle* h = new icc_handle();
  icc_default_solver_options(&h->opt);
  memset(&h->P, 0, sizeof h->P);
  *out = h;
  if (device_ordinal < 0) { h->device = -1; return ICC_OK; }
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0 || device_ordinal >= count) {
    h->err = std::string("no usable CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device ordinal out of range") + "); this library has no CPU fallback";
    return ICC_ERR_NO_DEVICE;
  }
  if (cudaSetDevice(device_ordinal) != cudaSuccess) { h->err = "cudaSetDevice failed"; return ICC_ERR_NO_DEVICE; }
  h->device = device_ordinal;
  cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device_ordinal);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { h->err = "cudaStreamCreate failed"; h->device = -1; return ICC_ERR_CUDA; }
  if (h->d_scal.alloc(SC_COUNT) != cudaSuccess) { h->err = "cudaMalloc failed"; return ICC_ERR_CUDA; }
  h->aux_ok = cudaStreamCreateWithFlags(&h->aux.stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&h->aux.fork, cudaEventDisableTiming) == cudaSuccess && cudaEventCreateWithFlags(&h->aux.join, cudaEventDisableTiming) == cudaSuccess;
  if (!h->aux_ok) { h->err = "cudaStreamCreate failed"; return ICC_ERR_CUDA; }
  return ICC_OK;
}
void icc_destroy(icc_handle* h) { if (!h) return; if (h->device >= 0) { cudaSetDevice(h->device); if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); } if (h->aux_ok) { cudaStreamDestroy(h->aux.stream); cudaEventDestroy(h->aux.fork); cudaEventDestroy(h->aux.join); } } delete h; }
const char* icc_last_error(const icc_handle* h) { return h ? h->err.c_str() : "null handle"; }
icc_status icc_set_solver_options(icc_handle* h, const icc_solver_options* o) { if (!h || !o) return ICC_ERR_INVALID_ARGUMENT; h->opt = *o; return ICC_OK; }

icc_status icc_set_camera(icc_handle* h, int model, const double* intr, int n, int w, int hgt) {
  if (!h || !intr) return ICC_ERR_INVALID_ARGUMENT;
  if (camera_num_params(model) < 0 || n != camera_num_params(model)) return fail(h, ICC_ERR_INVALID_ARGUMENT, "unknown camera model or wrong intrinsic count");
  h->model = model; h->n_intr = n; h->width = w; h->height = hgt; for (int i = 0; i < n; ++i) h->intr[i] = intr[i];
  return ICC_OK;
}
icc_status icc_set_board_points(icc_handle* h, int n, const double* xyzw) {
  if (!h || n <= 0 || !xyzw) return ICC_ERR_INVALID_ARGUMENT;
  const bool same_board = h->points.size() == 4 * (size_t)n;
  if (h->initialised && h->device >= 0 && same_board) { icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s; }
  h->points.assign(xyzw, xyzw + 4 * (size_t)n);
  if (h->initialised && h->device >= 0) {      // an assembled problem keeps its corners: only the coordinates may change
    if (!same_board) return fail(h, ICC_ERR_STATE, "the number of board points cannot change after batch_init_spline");
    for (int k = 0; k < 2; ++k) { icc_status s = upload_points(h, k, false); if (s != ICC_OK) return s; }
  }
  return ICC_OK;
}
icc_status icc_set_frames(icc_handle* h, int nf, const double* t, const int32_t* off, const int32_t* ids, const double* uv, const double* q, const double* p) {
  if (!h || nf <= 0 || !t || !off || !ids || !uv || !q || !p) return ICC_ERR_INVALID_ARGUMENT;
  const int nc = off[nf];
  for (int i = 0; i < nf; ++i) if (off[i + 1] < off[i]) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must be non-decreasing");
  if (h->device >= 0 && h->stream) cudaStreamSynchronize(h->stream);   // an asynchronous upload may still be reading the staging buffers
  const bool pin = h->device >= 0;
  h->frame_t.assign(t, t + nf); h->corner_off.assign(off, off + nf + 1);
  h->n_corners_in = (size_t)nc;
  h->frames_dev = pin && nc > 0 && host_is_pinned(uv) && host_is_pinned(ids);
  if (h->frames_dev) {   // page-locked caller buffers: DMA straight to the device, the id range is found while it runs
    CU(cudaSetDevice(h->device));
    CU(h->d_uv_all.alloc((size_t)nc)); CU(h->d_pid_all.alloc((size_t)nc));
    CU(cudaMemcpyAsync(h->d_uv_all.p, uv, (size_t)nc * sizeof(double2), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_pid_all.p, ids, (size_t)nc * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    // the id range is reduced on the device behind the copy (two ints come back with the synchronisation this call ends with anyway)
    int* rng = static_cast<int*>(h->arena_small(2 * sizeof(int)));
    if (rng) {
      rng[0] = 0; rng[1] = -1;
      CU(h->d_idrange.alloc(2));
      CU(cudaMemcpyAsync(h->d_idrange.p, rng, 2 * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      launch_id_range(nc, h->d_pid_all.p, h->d_idrange.p, h->stream);
      CU(cudaMemcpyAsync(rng, h->d_idrange.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    }
    h->uv.clear(); h->point_ids.clear();
    CU(cudaStreamSynchronize(h->stream));   // the caller's arrays are not referenced after this call returns
    if (rng) { h->id_lo = rng[0]; h->id_hi = rng[1]; }
    else { int lo = 0, hi = -1; for (int i = 0; i < nc; ++i) { const int v = ids[i]; lo = v < lo ? v : lo; hi = v > hi ? v : hi; } h->id_lo = lo; h->id_hi = hi; }
  } else {
    h->uv.assign(uv, 2 * (size_t)nc, pin);
    // the ids are copied and range-checked in one pass (the check of batch_init_spline would read them again, cold)
    h->point_ids.resize((size_t)nc, pin);
    int lo = 0, hi = -1; int* dst = h->point_ids.data();
    for (int i = 0; i < nc; ++i) { const int v = ids[i]; dst[i] = v; lo = v < lo ? v : lo; hi = v > hi ? v : hi; }
    h->id_lo = lo; h->id_hi = hi;
  }
  h->q_wc.assign(q, q + 4 * (size_t)nf); h->p_wc.assign(p, p + 3 * (size_t)nf);
  return ICC_OK;
}
icc_status icc_set_imu(icc_handle* h, int n, const double* t, const double* a, const double* g) {
  if (!h || n < 0 || (n > 0 && (!t || !a || !g))) return ICC_ERR_INVALID_ARGUMENT;
  if (h->device >= 0 && h->stream) cudaStreamSynchronize(h->stream);
  const bool pin = h->device >= 0;
  h->n_imu_in = (size_t)n;
  h->imu_dev = pin && n > 0 && host_is_pinned(a) && host_is_pinned(g);
  if (h->imu_dev) {
    CU(cudaSetDevice(h->device));
    CU(h->d_acc_all.alloc(3 * (size_t)n)); CU(h->d_gyr_all.alloc(3 * (size_t)n));
    CU(cudaMemcpyAsync(h->d_acc_all.p, a, 3 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_gyr_all.p, g, 3 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    h->imu_acc.clear(); h->imu_gyr.clear();
  } else { h->imu_acc.assign(a, 3 * (size_t)n, pin); h->imu_gyr.assign(g, 3 * (size_t)n, pin); }
  {   // time stamps: copied and tested for order in one pass (the sorted stream takes the bisection path of batch_init_spline)
    h->imu_t.resize((size_t)n, pin);
    double* dst = h->imu_t.data(); int unsorted = 0; double prev = n > 0 ? t[0] : 0.0;
    for (int i = 0; i < n; ++i) { const double v = t[i]; dst[i] = v; unsorted |= !(v >= prev); prev = v; }
    h->imu_sorted = !unsorted;
  }
  if (h->imu_dev) CU(cudaStreamSynchronize(h->stream));   // the caller's arrays are not referenced after this call returns
  return ICC_OK;
}
icc_status icc_set_shard(icc_handle* h, int rank, int world) { if (!h || world < 1 || rank < 0 || rank >= world) return fail(h, ICC_ERR_INVALID_ARGUMENT, "bad shard"); h->shard_rank = rank; h->shard_world = world; return ICC_OK; }
icc_status icc_set_comm(icc_handle* h, icc_comm* c) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  h->comm = c;
  h->shard_rank = c ? icc_comm_rank(c) : 0; h->shard_world = c ? icc_comm_world(c) : 1;
  return ICC_OK;
}
icc_status icc_set_allreduce(icc_handle* h, icc_allreduce_fn fn, void* user) { if (!h) return ICC_ERR_INVALID_ARGUMENT; h->allreduce = fn; h->allreduce_user = user; return ICC_OK; }

icc_status icc_set_bias_splines(icc_handle* h, double acc_dt_s, double gyr_dt_s) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  for (const double dt : {acc_dt_s, gyr_dt_s})   // <= 0 selects the reference's 10 s; a spacing must be a whole number of nanoseconds >= 1
    if (!std::isfinite(dt) || (dt > 0.0 && (dt * S_TO_NS < 1.0 || dt > 1e9)))
      return fail(h, ICC_ERR_INVALID_ARGUMENT, "bias knot spacing must be finite and either <= 0 (the default 10 s) or in [1 ns, 1e9 s]");
  h->bias_dt_s_set[0] = acc_dt_s; h->bias_dt_s_set[1] = gyr_dt_s;
  return ICC_OK;
}
icc_status icc_set_bias_random_walk(icc_handle* h, const double acc_q[3], const double gyr_q[3]) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  const double* q[2] = {acc_q, gyr_q};
  for (int s = 0; s < 2; ++s)
    if (q[s]) for (int a = 0; a < 3; ++a)
      if (!(q[s][a] > 0.0) || !std::isfinite(q[s][a])) return fail(h, ICC_ERR_INVALID_ARGUMENT, "random-walk densities must be finite and > 0 (NULL turns a sensor's prior off)");
  for (int s = 0; s < 2; ++s) { h->walk_set[s] = q[s] != nullptr; for (int a = 0; a < 3; ++a) h->walk_q_set[s][a] = q[s] ? q[s][a] : 0.0; }
  return ICC_OK;
}
icc_status icc_num_bias_prior_residuals(const icc_handle* h, int* n) { if (!h || !n) return ICC_ERR_INVALID_ARGUMENT; *n = h->n_res_prior; return ICC_OK; }

icc_status icc_batch_init_spline(icc_handle* h, const icc_init_params* ipp) {
  if (!h || !ipp) return ICC_ERR_INVALID_ARGUMENT;
  if (h->model < 0 || h->frame_t.empty() || h->points.empty()) return fail(h, ICC_ERR_STATE, "camera, board points and frames must be set before batch_init_spline");
  PhaseTrace trace(h->device >= 0 ? h->stream : nullptr);
  if (h->id_lo < 0 || (size_t)(h->id_hi + 1) > h->points.size() / 4) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner references an unknown board point");
  h->ip = *ipp;
  trace.lap("batch_init: id range check");
  KnotCounts n;
  icc_status s = init_globals_and_knot_counts(h, n); if (s != ICC_OK) return s;
  const ViewTable views = view_table(h);
  const Pose Tci = T_c_i(h);
  if (h->device < 0) init_knots_on_host(h, views, Tci);   // with a device, init_knots_kernel writes them straight into both state copies
  trace.lap("batch_init: ranges, view order, bias knots");
  // ---- measurement wiring (imu_camera_calibrator.cc:87-120; Add*Measurement impl.h:341-613) ----------------------
  std::vector<int> accepted, frame_sel;
  const std::vector<FrameHost> frames = frame_times(h, n, accepted);
  trace.lap("batch_init: frame times");
  if (!select_sorted(h, n, frames, accepted, views.increasing, frame_sel)) { s = select_general(h, n, frames, accepted, frame_sel); if (s != ICC_OK) return s; }
  trace.lap("batch_init: imu pass");
  s = gather_corners(h, frames, frame_sel); if (s != ICC_OK) return s;
  trace.lap("batch_init: host assembly");
  s = init_gravity(h, views, Tci); if (s != ICC_OK) return s;
  DeviceProblem& P = h->P;
  memset(&P, 0, sizeof P);
  P.model = h->model; P.dispatch_fov = ipp->dispatch_fov; P.n_intr = h->n_intr;
  P.n_frames = (int)h->frames.size(); P.n_corners = h->used_n; P.rolling = ipp->init_line_delay_s != 0.0 ? 1 : 0;
  P.n_imu = (int)h->n_imu_used; P.n_cells = (int)h->cells.size();
  P.dt_so3_ns = h->dt_so3_ns; P.dt_r3_ns = h->dt_r3_ns; P.dt_ba_ns = h->dt_ba_ns; P.dt_bg_ns = h->dt_bg_ns;
  P.inv_so3_dt = S_TO_NS / double(h->dt_so3_ns); P.inv_r3_dt = S_TO_NS / double(h->dt_r3_ns);
  P.w_acc = 1.0 / ipp->std_r3; P.w_gyr = 1.0 / ipp->std_so3;
  P.n_so3 = n.so3; P.n_r3 = n.r3; P.n_ba = n.ba; P.n_bg = n.bg;
  P.n_res_vis = P.rolling ? 2 * P.n_corners : 0; P.n_res_acc = 3 * P.n_imu; P.n_res_gyr = 3 * P.n_imu;
  const EvalStreams streams = eval_schedule(h);
  h->cur_flags = -1; h->ne_flags = -1; h->initialised = true; h->cur = 0; h->state_dirty_host = false; h->knots_dirty_host = false;
  if (h->device < 0) return ICC_OK;
  return upload_problem(h, views, Tci, streams, trace);
}

icc_status icc_set_known_gravity_dir(icc_handle* h, const double g[3]) {
  if (!h || !g) return ICC_ERR_INVALID_ARGUMENT;
  if (h->state_dirty_host) { icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s; }   // (knots alone being newer on the device does not matter here)
  for (int d = 0; d < 3; ++d) h->glob[G_GRAV + d] = g[d];
  if (h->device >= 0 && h->initialised) {   // only the globals block changed: one small staged copy instead of the whole state
    CU(cudaSetDevice(h->device));
    CU(upload_staged(h, h->st[h->cur].glob, std::vector<double>(h->glob, h->glob + G_COUNT)));
    return ICC_OK;
  }
  return push_state_to_device(h);
}

icc_status icc_optimize(icc_handle* h, int max_iterations, int flags, icc_summary* summary) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  icc_summary S;
  icc_status s = run_lm(h, max_iterations, flags, true, &S); if (s != ICC_OK) return s;
  const int l0 = kernel_launch_count();
  PhaseTrace trace(h->stream);
  s = mean_reproj(h, &S.mean_reproj_error); if (s != ICC_OK) return s;
  trace.lap("optimize: mean reprojection error");
  S.gpu_launches += kernel_launch_count() - l0;
  if (summary) *summary = S;
  return ICC_OK;
}
icc_status icc_lm_iterations(icc_handle* h, int n, int flags, icc_summary* summary) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  return run_lm(h, n, flags, false, summary);
}

icc_status icc_get_T_i_c(const icc_handle* hc, double T[7]) { icc_handle* h = const_cast<icc_handle*>(hc); if (!h || !T) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_globals_to_host(h); if (s != ICC_OK) return s; memcpy(T, h->glob + G_TIC, 7 * sizeof(double)); return ICC_OK; }
icc_status icc_get_gravity(const icc_handle* hc, double g[3]) { icc_handle* h = const_cast<icc_handle*>(hc); if (!h || !g) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_globals_to_host(h); if (s != ICC_OK) return s; memcpy(g, h->glob + G_GRAV, 3 * sizeof(double)); return ICC_OK; }
icc_status icc_get_line_delay(const icc_handle* hc, double* ld) { icc_handle* h = const_cast<icc_handle*>(hc); if (!h || !ld) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_globals_to_host(h); if (s != ICC_OK) return s; *ld = h->glob[G_LD]; return ICC_OK; }
icc_status icc_get_camera_intrinsics(const icc_handle* hc, double* k, int n) { icc_handle* h = const_cast<icc_handle*>(hc); if (!h || !k) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_globals_to_host(h); if (s != ICC_OK) return s; for (int i = 0; i < n && i < h->n_intr; ++i) k[i] = h->initialised ? h->glob[G_CAM_INTR + i] : h->intr[i]; return ICC_OK; }
icc_status icc_get_time_offset(const icc_handle* hc, double* t) { icc_handle* h = const_cast<icc_handle*>(hc); if (!h || !t) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_globals_to_host(h); if (s != ICC_OK) return s; *t = h->ip.time_offset_imu_to_cam_s + h->glob[G_TOFF]; return ICC_OK; }
icc_status icc_get_num_knots(const icc_handle* h, int* a, int* b, int* c, int* d) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (a) *a = (int)h->so3.size() / 4; if (b) *b = (int)h->r3.size() / 3; if (c) *c = (int)h->ba.size() / 3; if (d) *d = (int)h->bg.size() / 3;
  return ICC_OK;
}
icc_status icc_get_knots(const icc_handle* hc, double* so3, double* r3, double* ba, double* bg) {
  icc_handle* h = const_cast<icc_handle*>(hc); if (!h) return ICC_ERR_INVALID_ARGUMENT;
  icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s;
  if (so3) std::copy(h->so3.begin(), h->so3.end(), so3);
  if (r3) std::copy(h->r3.begin(), h->r3.end(), r3);
  if (ba) std::copy(h->ba.begin(), h->ba.end(), ba);
  if (bg) std::copy(h->bg.begin(), h->bg.end(), bg);
  return ICC_OK;
}
icc_status icc_set_knots(icc_handle* h, const double* so3, const double* r3, const double* ba, const double* bg) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s;
  if (so3) std::copy(so3, so3 + h->so3.size(), h->so3.begin());
  if (r3) std::copy(r3, r3 + h->r3.size(), h->r3.begin());
  if (ba) std::copy(ba, ba + h->ba.size(), h->ba.begin());
  if (bg) std::copy(bg, bg + h->bg.size(), h->bg.begin());
  return push_state_to_device(h);
}
icc_status icc_set_T_i_c(icc_handle* h, const double T[7]) { if (!h || !T) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s; memcpy(h->glob + G_TIC, T, 7 * sizeof(double)); return push_state_to_device(h); }
icc_status icc_set_line_delay(icc_handle* h, double ld) { if (!h) return ICC_ERR_INVALID_ARGUMENT; icc_status s = sync_state_to_host(h); if (s != ICC_OK) return s; h->glob[G_LD] = ld; return push_state_to_device(h); }
icc_status icc_get_mean_reprojection_error(icc_handle* h, double* e) {
  if (!h || !e) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  return mean_reproj(h, e);
}
icc_status icc_get_num_imu_cells(const icc_handle* h, int* n) { if (!h || !n) return ICC_ERR_INVALID_ARGUMENT; *n = (int)h->cells.size(); return ICC_OK; }
icc_status icc_get_imu_cells(const icc_handle* h, int32_t* c6) {
  if (!h || !c6) return ICC_ERR_INVALID_ARGUMENT;
  for (size_t k = 0; k < h->cells.size(); ++k) { const ImuCell& c = h->cells[k]; int32_t* o = c6 + 6 * k; o[0] = c.s_so3; o[1] = c.s_r3; o[2] = c.s_ba; o[3] = c.s_bg; o[4] = c.i_begin; o[5] = c.i_end; }
  return ICC_OK;
}
icc_status icc_get_eval_schedule(const icc_handle* h, int32_t counts4[4], int32_t* vitems3, int32_t* iitems3) {
  if (!h || !counts4) return ICC_ERR_INVALID_ARGUMENT;
  if (!h->initialised) return ICC_ERR_STATE;
  counts4[0] = h->P.n_vchunks; counts4[1] = h->P.n_ichunks; counts4[2] = (int32_t)h->vitems.size(); counts4[3] = (int32_t)h->iitems.size();
  for (int s = 0; s < 2; ++s) {
    int32_t* o = s ? iitems3 : vitems3;
    if (!o) continue;
    for (const VisItem& it : s ? h->iitems : h->vitems) { o[0] = it.vf0; o[1] = it.pos_begin; o[2] = it.pos_end; o += 3; }
  }
  return ICC_OK;
}
icc_status icc_get_num_imu_used(const icc_handle* h, int* n) { if (!h || !n) return ICC_ERR_INVALID_ARGUMENT; *n = (int)h->n_imu_used; return ICC_OK; }
icc_status icc_get_imu_used(const icc_handle* hc, double* t, double* a, double* g) {
  icc_handle* h = const_cast<icc_handle*>(hc);
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (a || g) { icc_status es = ensure_host_imu(h); if (es != ICC_OK) return es; }
  const size_t nu = h->n_imu_used;
  if (t) { if (h->imu_lazy) { for (size_t k = 0; k < nu; ++k) t[k] = h->imu_t[h->imu_src0 + k] + h->ip.time_offset_imu_to_cam_s; } else std::copy(h->imu_used_t.begin(), h->imu_used_t.end(), t); }
  if (a) { const double* src = h->imu_contig ? h->imu_acc.data() + 3 * (size_t)h->imu_src0 : h->imu_used_acc.data(); std::copy(src, src + 3 * nu, a); }
  if (g) { const double* src = h->imu_contig ? h->imu_gyr.data() + 3 * (size_t)h->imu_src0 : h->imu_used_gyr.data(); std::copy(src, src + 3 * nu, g); }
  return ICC_OK;
}

icc_status icc_eval_trajectory(icc_handle* h, int n, const int64_t* t_ns, double* gyro, double* accel, double* gb, double* ab, double* pq, double* pp, int32_t* valid) {
  if (!h || n < 0 || (n > 0 && !t_ns)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  if (n == 0) return ICC_OK;
  CU(cudaSetDevice(h->device));
  DevBuf<int64_t> d_t; DevBuf<double> d_out; DevBuf<int> d_valid;
  std::vector<int64_t> tv(t_ns, t_ns + n);
  CU(d_t.upload(tv)); CU(d_out.alloc((size_t)n * 19)); CU(d_valid.alloc(n));
  CU(cudaMemsetAsync(d_out.p, 0, (size_t)n * 19 * sizeof(double), h->stream));
  double* o = d_out.p;
  launch_eval_trajectory(h->P, h->st[h->cur].view(), n, d_t.p, h->start_ns, o, o + 3 * n, o + 6 * n, o + 9 * n, o + 12 * n, o + 16 * n, d_valid.p, h->stream);
  std::vector<double> ho((size_t)n * 19); std::vector<int> hv(n);
  CU(cudaMemcpyAsync(ho.data(), d_out.p, ho.size() * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(hv.data(), d_valid.p, n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < n; ++i) {
    const bool v = hv[i] != 0;
    if (valid) valid[i] = hv[i];
    // like the reference getters, outputs are only written where CalcTimes accepts the timestamp (gyro needs SO3 only,
    // but the hot CLI queries inside the spline range where both hold)
    if (gyro && v) for (int d = 0; d < 3; ++d) gyro[3 * i + d] = ho[3 * i + d];
    if (accel && v) for (int d = 0; d < 3; ++d) accel[3 * i + d] = ho[3 * n + 3 * i + d];
    if (gb) for (int d = 0; d < 3; ++d) gb[3 * i + d] = ho[6 * n + 3 * i + d];
    if (ab) for (int d = 0; d < 3; ++d) ab[3 * i + d] = ho[9 * n + 3 * i + d];
    if (pq && v) for (int d = 0; d < 4; ++d) pq[4 * i + d] = ho[12 * n + 4 * i + d];
    if (pp && v) for (int d = 0; d < 3; ++d) pp[3 * i + d] = ho[16 * n + 3 * i + d];
  }
  return ICC_OK;
}

icc_status icc_num_residuals(const icc_handle* h, int* v, int* a, int* g) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (v) *v = h->P.n_res_vis; if (a) *a = h->P.n_res_acc; if (g) *g = h->P.n_res_gyr;
  return ICC_OK;
}
icc_status icc_num_tangent(const icc_handle* hc, int flags, int* n) {
  icc_handle* h = const_cast<icc_handle*>(hc);
  if (!h || !n) return ICC_ERR_INVALID_ARGUMENT;
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  icc_status s = configure(h, flags); if (s != ICC_OK) return s;
  *n = h->n_tan; return ICC_OK;
}

icc_status icc_evaluate(icc_handle* h, int flags, double* cost, double* residuals, double* gradient, double* hessian) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  icc_status s = configure(h, flags); if (s != ICC_OK) return s;
  const DeviceProblem& P = h->P;
  const int nres = P.n_res_vis + P.n_res_acc + P.n_res_gyr + h->n_res_prior, n = h->n_tan;
  double* res_dev = nullptr;
  if (residuals) { CU(h->d_res.alloc((size_t)std::max(1, nres))); CU(cudaMemsetAsync(h->d_res.p, 0, (size_t)nres * sizeof(double), h->stream)); res_dev = h->d_res.p; }
  if (!gradient && !hessian) {
    CU(cudaMemsetAsync(h->d_scal.p, 0, SC_COUNT * sizeof(double), h->stream));
    s = eval_cost(h, h->st[h->cur].view(), h->d_scal.p + SC_CAND_COST, res_dev, nullptr); if (s != ICC_OK) return s;
    double c; CU(cudaMemcpyAsync(&c, h->d_scal.p + SC_CAND_COST, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (residuals) CU(cudaMemcpyAsync(residuals, res_dev, (size_t)nres * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    if (cost) *cost = c;
    return ICC_OK;
  }
  s = eval_jacobian(h, h->st[h->cur].view(), res_dev); if (s != ICC_OK) return s;
  std::vector<double> ne((size_t)P.ne_size);
  CU(cudaMemcpyAsync(ne.data(), P.ne, ne.size() * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (residuals) CU(cudaMemcpyAsync(residuals, res_dev, (size_t)nres * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  h->ne_flags = flags;
  if (cost) *cost = ne[P.ne_off_cost];
  if (gradient) for (int i = 0; i < n; ++i) gradient[i] = ne[P.ne_off_g + h->perm[i]];
  if (hessian) {
    auto get = [&](int a, int b) -> double {
      const int lo = std::min(a, b), hi = std::max(a, b);
      if (hi < P.nk) return hi - lo <= P.kd ? ne[(size_t)lo * P.ldb + (hi - lo)] : 0.0;
      if (lo < P.nk) return ne[P.ne_off_E + (size_t)lo * P.nb + (hi - P.nk)];
      return ne[P.ne_off_C + (size_t)(hi - P.nk) * P.nb + (lo - P.nk)];
    };
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) hessian[(size_t)i * n + j] = get(h->perm[i], h->perm[j]);
  }
  return ICC_OK;
}

// J^T J products with caller-supplied vectors (canonical tangent order, nvec columns stored one after the other): the packed
// banded + bordered normal equations are read back once and multiplied on the host.  Evaluation / parity helper: a dense Hessian of
// BASELINE config 4 would be 1.2 GB, a handful of products check every stored entry of J^T J at full size.
icc_status icc_normal_matvec(icc_handle* h, int flags, int nvec, const double* V, double* HV) {
  if (!h || nvec <= 0 || !V || !HV) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  icc_status s = configure(h, flags); if (s != ICC_OK) return s;
  const DeviceProblem& P = h->P;
  const int n = h->n_tan, nk = P.nk, nb = P.nb;
  s = eval_jacobian(h, h->st[h->cur].view(), nullptr); if (s != ICC_OK) return s;
  std::vector<double> ne((size_t)P.ne_size);
  CU(cudaMemcpyAsync(ne.data(), P.ne, ne.size() * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  std::vector<double> x((size_t)n), y((size_t)n);
  for (int v = 0; v < nvec; ++v) {
    for (int i = 0; i < n; ++i) x[h->perm[i]] = V[(size_t)v * n + i];
    std::fill(y.begin(), y.end(), 0.0);
    for (int lo = 0; lo < nk; ++lo) {
      const double* col = &ne[(size_t)lo * P.ldb];
      y[lo] += col[0] * x[lo];
      for (int d = 1; d <= P.kd && lo + d < nk; ++d) { y[lo] += col[d] * x[lo + d]; y[lo + d] += col[d] * x[lo]; }
      const double* e = &ne[P.ne_off_E + (size_t)lo * nb];
      for (int b = 0; b < nb; ++b) { y[lo] += e[b] * x[nk + b]; y[nk + b] += e[b] * x[lo]; }
    }
    for (int hi = 0; hi < nb; ++hi) for (int lo = 0; lo <= hi; ++lo) {
      const double c = ne[P.ne_off_C + (size_t)hi * nb + lo];
      y[nk + hi] += c * x[nk + lo]; if (lo != hi) y[nk + lo] += c * x[nk + hi];
    }
    for (int i = 0; i < n; ++i) HV[(size_t)v * n + i] = y[h->perm[i]];
  }
  h->ne_flags = flags;
  return ICC_OK;
}

int64_t icc_kernel_launch_count(void) { return kernel_launch_count(); }

icc_status icc_solver_plan(icc_handle* h, int flags, int chunks, icc_solver_plan_info* plan) {
  if (!h || !plan || chunks < 0) return ICC_ERR_INVALID_ARGUMENT;
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  if (h->device >= 0) CU(cudaSetDevice(h->device));
  icc_status s = configure(h, flags); if (s != ICC_OK) return s;
  solver_plan_info(h->P, chunks, plan);
  return ICC_OK;
}

// The linear solve of one LM iteration on the normal equations already in the handle: what run_lm launches between the Jacobian
// and the update, with the plan's own workspace, so that a test can compare the step with a dense solve of exactly the H and g
// that were factored.
icc_status icc_solve_normal_equations(icc_handle* h, int flags, double radius, int chunks, double* delta, double* scale, double* h_diag,
                                      double* model_change, int32_t* step_ok, icc_solver_plan_info* plan) {
  if (!h || chunks < 0 || !(radius > 0.0)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  if (h->ne_flags != flags || h->cur_flags != flags)
    return fail(h, ICC_ERR_STATE, "no current normal equations for these flags: call icc_evaluate (gradient or Hessian) or icc_normal_matvec first");
  CU(cudaSetDevice(h->device));
  const DeviceProblem& P = h->P;
  const int n = P.nk + P.nb;
  icc_solver_plan_info pi; solver_plan_info(P, chunks, &pi);
  if (plan) *plan = pi;
  if (!pi.valid) return fail(h, ICC_ERR_UNSUPPORTED, border_too_wide_message(h));
  if (n == 0) { if (model_change) *model_change = 0.0; if (step_ok) *step_ok = 1; return ICC_OK; }
  DevBuf<double> ws; CU(ws.alloc((size_t)pi.workspace_doubles));
  CU(cudaMemsetAsync(h->d_scal.p, 0, SC_COUNT * sizeof(double), h->stream));
  launch_compute_scale(P, h->d_scale.p, h->opt.jacobi_scaling, h->d_scal.p, h->stream);
  SolveParams sp; sp.radius = radius; sp.min_diag = h->opt.min_lm_diagonal; sp.max_diag = h->opt.max_lm_diagonal; sp.jacobi_scaling = h->opt.jacobi_scaling;
  const int se = launch_solve(P, h->d_scale.p, sp, ws.p, h->d_delta.p, h->d_scal.p, h->stream, chunks);
  if (se) return fail(h, ICC_ERR_CUDA, std::string("solver launch: ") + cudaGetErrorString(cudaGetLastError()));
  std::vector<double> d(n), s(n), hd(n); double sc[SC_COUNT];
  CU(cudaMemcpyAsync(d.data(), h->d_delta.p, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(s.data(), h->d_scale.p, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (P.nk) CU(cudaMemcpy2DAsync(hd.data(), sizeof(double), P.ne, (size_t)P.ldb * sizeof(double), sizeof(double), P.nk, cudaMemcpyDeviceToHost, h->stream));
  if (P.nb) CU(cudaMemcpy2DAsync(hd.data() + P.nk, sizeof(double), P.ne + P.ne_off_C, (size_t)(P.nb + 1) * sizeof(double), sizeof(double), P.nb, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(sc, h->d_scal.p, sizeof sc, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  const bool ok = sc[SC_OK] == 1.0;
  for (int i = 0; i < n; ++i) {
    const int k = h->perm[i];
    if (delta && ok) delta[i] = d[k];
    if (scale) scale[i] = s[k];
    if (h_diag) h_diag[i] = hd[k];
  }
  if (model_change) *model_change = sc[SC_MODEL_CHANGE];
  if (step_ok) *step_ok = ok ? 1 : 0;
  return ICC_OK;
}

icc_status icc_time_evaluations(icc_handle* h, int n, int flags, int with_jacobian, double* ms_per_eval) {
  if (!h || !ms_per_eval || n <= 0) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  icc_status s = configure(h, flags); if (s != ICC_OK) return s;
  h->ne_flags = -1;                        // the single-family modes accumulate into the normal equations without zeroing them
  cudaEvent_t e0, e1; CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
  CU(cudaMemsetAsync(h->d_scal.p, 0, SC_COUNT * sizeof(double), h->stream));
  CU(cudaEventRecord(e0, h->stream));
  for (int i = 0; i < n; ++i) {
    if (with_jacobian == 1) { s = eval_jacobian(h, h->st[h->cur].view(), nullptr); }
    else if (with_jacobian == 2 || with_jacobian == 3) {   // one kernel family only (2 = vision, 3 = imu), Jacobian mode, no memset
      DeviceProblem Q = h->P; if (with_jacobian == 2) Q.n_iwork = 0; else { Q.n_vwork = 0; Q.n_vitems = 0; }
      if (with_jacobian == 2) Q.n_iitems = 0;
      s = launch_eval(Q, h->st[h->cur].view(), true, nullptr, nullptr, nullptr, h->stream, nullptr, tangent_meas(h)) ? fail(h, ICC_ERR_CUDA, "eval launch failed") : ICC_OK;
    }
    else { s = eval_cost(h, h->st[h->cur].view(), h->d_scal.p + SC_CAND_COST, nullptr, nullptr); }
    if (s != ICC_OK) return s;
  }
  CU(cudaEventRecord(e1, h->stream));
  CU(cudaEventSynchronize(e1));
  float ms = 0; CU(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms_per_eval = ms / n;
  return ICC_OK;
}

void* icc_get_stream(icc_handle* h) { return h ? (void*)h->stream : nullptr; }
// ---- upstream row f1: per-view board poses (icc_pose.cu) ----------------------------------------------------------------
icc_status icc_pixels_to_normalized(icc_handle* h, int n, const double* uv, double* xy_out, int32_t* ok) {
  if (!h || n < 0 || (n > 0 && (!uv || !xy_out))) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (h->model < 0) return fail(h, ICC_ERR_STATE, "icc_set_camera must be called first");
  if (n == 0) return ICC_OK;
  return drive(h, [&](std::string& err) { return pixels_to_normalized(h->stream, h->model, h->intr, n, uv, xy_out, ok, err); });
}

icc_status icc_pixels_to_bearings(icc_handle* h, int n, const double* uv, double* xyz_out, int32_t* ok) {
  if (!h || n < 0 || (n > 0 && (!uv || !xyz_out))) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (h->model < 0) return fail(h, ICC_ERR_STATE, "icc_set_camera must be called first");
  if (n == 0) return ICC_OK;
  return drive(h, [&](std::string& err) { return pixels_to_bearings(h->stream, h->model, h->intr, n, uv, xyz_out, ok, err); });
}

icc_status icc_set_reprojection_error(icc_handle* h, int mode) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (h->initialised) return fail(h, ICC_ERR_STATE, "the reprojection error must be chosen before icc_batch_init_spline");
  if (mode != ICC_REPROJ_ERROR_PIXEL && mode != ICC_REPROJ_ERROR_TANGENT) return fail(h, ICC_ERR_INVALID_ARGUMENT, "reprojection error must be ICC_REPROJ_ERROR_PIXEL (0) or ICC_REPROJ_ERROR_TANGENT (1)");
  h->reproj_error = mode;
  return ICC_OK;
}

icc_status icc_set_pose_error(icc_handle* h, int mode) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (mode != ICC_POSE_ERROR_NORMALIZED && mode != ICC_POSE_ERROR_TANGENT) return fail(h, ICC_ERR_INVALID_ARGUMENT, "pose error must be ICC_POSE_ERROR_NORMALIZED (0) or ICC_POSE_ERROR_TANGENT (1)");
  h->pose_error = mode;
  return ICC_OK;
}

icc_status icc_set_pose_rolling_shutter(icc_handle* h, double line_delay_s, int32_t n_frames, const double* frame_t_s) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (!std::isfinite(line_delay_s) || line_delay_s < 0.0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "line delay must be finite and >= 0");
  if (line_delay_s == 0.0) { h->pose_line_delay = 0.0; h->pose_frame_t.clear(); return ICC_OK; }
  if (n_frames <= 0 || !frame_t_s) return fail(h, ICC_ERR_INVALID_ARGUMENT, "a rolling shutter needs the n_frames > 0 view times");
  for (int i = 0; i < n_frames; ++i)
    if (!std::isfinite(frame_t_s[i]) || frame_t_s[i] < 0.0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "view times must be finite and >= 0");
  h->pose_line_delay = line_delay_s;
  h->pose_frame_t.assign(frame_t_s, frame_t_s + n_frames);
  return ICC_OK;
}

icc_status icc_get_pose_velocities(const icc_handle* h, int32_t n_frames, double* w_u, int32_t* n_without_neighbours) {
  if (!h || n_frames <= 0 || !w_u) return ICC_ERR_INVALID_ARGUMENT;
  if (h->pose_vel.empty()) return fail(const_cast<icc_handle*>(h), ICC_ERR_STATE, "no rolling-shutter pose call has run on this handle");
  if ((size_t)n_frames * 6 != h->pose_vel.size()) return fail(const_cast<icc_handle*>(h), ICC_ERR_INVALID_ARGUMENT, "n_frames differs from the last rolling-shutter pose call");
  std::copy(h->pose_vel.begin(), h->pose_vel.end(), w_u);
  if (n_without_neighbours) *n_without_neighbours = h->pose_n_static;
  return ICC_OK;
}

// The shutter of the next pose call of nf views; its velocity outputs land in vel / n_static, which keep_velocities moves into the handle
// once the call has succeeded (a failed call leaves icc_get_pose_velocities as it was).  false (with the error set) when the view times of
// icc_set_pose_rolling_shutter are for another number of views.
struct PoseCallShutter {
  PoseShutter S; std::vector<double> vel; int32_t n_static = 0;
  bool prepare(icc_handle* h, int nf) {
    if (h->pose_line_delay <= 0.0) return true;
    if ((int)h->pose_frame_t.size() != nf) { fail(h, ICC_ERR_INVALID_ARGUMENT, "n_frames differs from the view times of icc_set_pose_rolling_shutter"); return false; }
    vel.assign(6 * (size_t)nf, 0.0);
    S.line_delay = h->pose_line_delay; S.frame_t = h->pose_frame_t.data(); S.vel = vel.data(); S.n_static = &n_static;
    return true;
  }
  icc_status keep_velocities(icc_handle* h, icc_status rc) {
    if (rc == ICC_OK && S.line_delay > 0.0) { h->pose_vel.swap(vel); h->pose_n_static = n_static; }
    return rc;
  }
};

icc_status icc_estimate_board_poses(icc_handle* h, int nf, const int32_t* off, const int32_t* ids, const double* uv, double max_reproj_error, int min_points, double* q_wc, double* p_wc, double* mean_err, int32_t* valid) {
  if (!h || nf <= 0 || !off || !ids || !uv || !q_wc || !p_wc || !valid) return ICC_ERR_INVALID_ARGUMENT;
  PoseCallShutter R;
  if (!R.prepare(h, nf)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (h->model < 0 || h->points.empty()) return fail(h, ICC_ERR_STATE, "icc_set_camera and icc_set_board_points must be called first");
  for (int i = 0; i < nf; ++i) if (off[i + 1] < off[i]) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must be non-decreasing");
  if (off[0] != 0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must start at 0");
  return R.keep_velocities(h, drive(h, [&](std::string& err) { return estimate_board_poses(h->stream, h->model, h->intr, h->width, h->height, (int)(h->points.size() / 4), h->points.data(), nf, off, ids, uv,
                                max_reproj_error, min_points, h->pose_error, R.S, q_wc, p_wc, mean_err, valid, err); }));
}

icc_status icc_filter_bad_poses(icc_handle* h, int nv, const double* p_wc, int32_t* valid) {
  if (nv <= 0 || !p_wc || !valid) return ICC_ERR_INVALID_ARGUMENT;
  filter_bad_poses(nv, p_wc, valid);
  return ICC_OK;
}

icc_status icc_get_board_points(const icc_handle* h, double* xyzw, int n) {
  if (!h || !xyzw || n < 0) return ICC_ERR_INVALID_ARGUMENT;
  { icc_status s = sync_state_to_host(const_cast<icc_handle*>(h)); if (s != ICC_OK) return s; }   // POINTS: the optimised points live in the device state
  const size_t m = std::min<size_t>(4 * (size_t)n, h->points.size());
  std::copy(h->points.begin(), h->points.begin() + m, xyzw);
  return ICC_OK;
}

icc_status icc_optimize_board_points(icc_handle* h, int nf, const int32_t* off, const int32_t* ids, const double* uv, double max_reproj_error, int min_points,
                                     int min_observations, double* q_wc, double* p_wc, double* mean_err, int32_t* valid, double* board_out, int32_t* n_opt_out) {
  if (!h || nf <= 0 || !off || !ids || !uv || !q_wc || !p_wc || !valid) return ICC_ERR_INVALID_ARGUMENT;
  PoseCallShutter R;
  if (!R.prepare(h, nf)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (h->model < 0 || h->points.empty()) return fail(h, ICC_ERR_STATE, "icc_set_camera and icc_set_board_points must be called first");
  if (off[0] != 0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must start at 0");
  for (int i = 0; i < nf; ++i) if (off[i + 1] < off[i]) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must be non-decreasing");
  std::vector<double> points;
  const icc_status rc = drive(h, [&](std::string& err) { return optimize_board_points(h->stream, h->model, h->intr, h->width, h->height, (int)(h->points.size() / 4), h->points.data(), nf, off, ids, uv, max_reproj_error, min_points,
                                 min_observations, h->pose_error, R.S, q_wc, p_wc, mean_err, valid, points, n_opt_out, err); });
  if (R.keep_velocities(h, rc) != ICC_OK) return rc;
  h->points.swap(points);
  if (board_out) std::copy(h->points.begin(), h->points.end(), board_out);
  return ICC_OK;
}

// ---- upstream row f3: IMU-to-camera rotation + time offset initialiser (icc_rotinit.cu) --------------------------------------
icc_status icc_estimate_imu_to_camera_rotation(icc_handle* h, int n_views, const double* view_t, const double* q_cw, int n_imu, const double* imu_t,
                                               const double* gyro, const double* bias_in, double* q_out, double* td_out, double* bias_out, double* err_out, int32_t* iters_out) {
  if (!h || n_views < 2 || !view_t || !q_cw || n_imu < 2 || !imu_t || !gyro || !q_out || !td_out) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  return drive(h, [&](std::string& err) { return estimate_imu_to_camera_rotation(h->stream, h->sm_count, n_views, view_t, q_cw, n_imu, imu_t, gyro, bias_in, q_out, td_out, bias_out, err_out, iters_out, err); });
}

// ---- upstream row f2: spline error weighting (icc_sew.cu) -----------------------------------------------------------------------
icc_status icc_spline_error_weighting(icc_handle* h, int n, const double* times, const double* signal, double quality, double min_dt, double max_dt, double* dt_out, double* var_out, double* spectrum) {
  if (!h || n < 4 || !times || !signal || !dt_out || !var_out || !(quality > 0.0 && quality < 1.0)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  return drive(h, [&](std::string& err) { return spline_error_weighting(h->stream, h->sm_count, n, times, signal, quality, min_dt, max_dt, dt_out, var_out, spectrum, err); });
}

// ---- upstream row f4: camera intrinsic calibration (icc_camcal.cu) ------------------------------------------------------------
icc_status icc_calibrate_camera(icc_handle* h, int model, int W, int H, int nv, const int32_t* off, const int32_t* ids, const double* uv,
                                const double* q_init, const double* p_init, const int32_t* init_valid, double focal_init, double distortion_init,
                                const icc_camcal_options* options, double* intr_out, double* q_out, double* p_out, double* err_out, int32_t* used_out, icc_camcal_summary* summary) {
  if (!h || nv <= 0 || !off || !ids || !uv || !intr_out || !q_out || !p_out || !used_out || W <= 0 || H <= 0) return ICC_ERR_INVALID_ARGUMENT;
  if (h->camcal_line_delay > 0.0 && nv != h->camcal_n_views) return fail(h, ICC_ERR_INVALID_ARGUMENT, "n_views differs from that of icc_set_camcal_rolling_shutter");
  NEED_DEVICE();
  if (camera_num_params(model) < 0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "unknown camera model");
  if (h->points.empty()) return fail(h, ICC_ERR_STATE, "icc_set_board_points must be called first");
  if (off[0] != 0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must start at 0");
  for (int i = 0; i < nv; ++i) if (off[i + 1] < off[i]) return fail(h, ICC_ERR_INVALID_ARGUMENT, "corner offsets must be non-decreasing");
  const int np = (int)(h->points.size() / 4);
  for (int i = 0; i < off[nv]; ++i) if (ids[i] < 0 || ids[i] >= np) return fail(h, ICC_ERR_INVALID_ARGUMENT, "point id outside the board");
  const bool rolling = h->camcal_line_delay > 0.0;
  std::vector<double> points; icc_camcal_summary S;
  std::vector<double> vel; int32_t n_static = 0;
  const icc_status rc = drive(h, [&](std::string& err) {
    auto calibrate = [&](const CamCalShutter& shutter) {
      points.clear();
      return calibrate_camera(h->stream, model, W, H, np, h->points.data(), nv, off, ids, uv, q_init, p_init, init_valid, focal_init, distortion_init, options,
                              intr_out, q_out, p_out, err_out, used_out, S, points, err, shutter);
    };
    if (!rolling) return calibrate(CamCalShutter{});
    if (!h->camcal_w_u.empty()) { vel = h->camcal_w_u; return calibrate(CamCalShutter{h->camcal_line_delay, vel.data()}); }
    // automatic mode: global-shutter round 0, then two rounds of (rolling-shutter pose step under the last intrinsics, calibration)
    icc_status r = calibrate(CamCalShutter{}); if (r != ICC_OK || !S.success) return r;
    std::vector<double> q(4 * (size_t)nv), p(3 * (size_t)nv), intr(MAX_INTR);
    std::vector<int32_t> valid(nv);
    vel.assign(6 * (size_t)nv, 0.0);
    for (int round = 1; round <= 2; ++round) {
      std::copy(intr_out, intr_out + std::max(10, camera_num_params(model)), intr.begin());
      const PoseShutter ps{h->camcal_line_delay, h->camcal_frame_t.data(), vel.data(), &n_static};
      r = estimate_board_poses(h->stream, model, intr.data(), W, H, np, h->points.data(), nv, off, ids, uv, 0.0, 0, h->pose_error, ps, q.data(), p.data(), nullptr, valid.data(), err);
      if (r != ICC_OK) return r;
      for (int i = 0; i < nv; ++i) if (!valid[i]) std::fill(vel.begin() + 6 * (size_t)i, vel.begin() + 6 * (size_t)i + 6, 0.0);
      r = calibrate(CamCalShutter{h->camcal_line_delay, vel.data()}); if (r != ICC_OK) return r;
    }
    return ICC_OK;
  });
  if (!points.empty()) h->points.swap(points);   // the board was refined, even if the final bundle adjustment then failed
  if (rc != ICC_OK) return rc;
  if (rolling && !vel.empty()) { h->camcal_vel.swap(vel); h->camcal_n_static = n_static; }
  if (summary) *summary = S;
  if (!S.success) h->err = "Not enough views for proper calibration";   // camera_calibrator.cc:132-135, :176-179, :202-205
  return ICC_OK;
}

icc_status icc_set_camcal_rolling_shutter(icc_handle* h, double line_delay_s, int32_t n_views, const double* frame_t_s, const double* w_u) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (!std::isfinite(line_delay_s) || line_delay_s < 0.0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "line delay must be finite and >= 0");
  if (line_delay_s == 0.0) { h->camcal_line_delay = 0.0; h->camcal_n_views = 0; h->camcal_frame_t.clear(); h->camcal_w_u.clear(); return ICC_OK; }
  if (n_views <= 0 || (!frame_t_s && !w_u)) return fail(h, ICC_ERR_INVALID_ARGUMENT, "a rolling shutter needs n_views > 0 and the view times or the view velocities");
  if (frame_t_s)
    for (int i = 0; i < n_views; ++i)
      if (!std::isfinite(frame_t_s[i]) || frame_t_s[i] < 0.0) return fail(h, ICC_ERR_INVALID_ARGUMENT, "view times must be finite and >= 0");
  if (w_u)
    for (size_t i = 0; i < 6 * (size_t)n_views; ++i) if (!std::isfinite(w_u[i])) return fail(h, ICC_ERR_INVALID_ARGUMENT, "view velocities must be finite");
  h->camcal_line_delay = line_delay_s; h->camcal_n_views = n_views;
  if (frame_t_s) h->camcal_frame_t.assign(frame_t_s, frame_t_s + n_views); else h->camcal_frame_t.clear();
  if (w_u) h->camcal_w_u.assign(w_u, w_u + 6 * (size_t)n_views); else h->camcal_w_u.clear();
  return ICC_OK;
}

icc_status icc_get_camcal_velocities(const icc_handle* h, int32_t n_views, double* w_u, int32_t* n_without_neighbours) {
  if (!h || n_views <= 0 || !w_u) return ICC_ERR_INVALID_ARGUMENT;
  if (h->camcal_vel.empty()) return fail(const_cast<icc_handle*>(h), ICC_ERR_STATE, "no rolling-shutter camera calibration has run on this handle");
  if ((size_t)n_views * 6 != h->camcal_vel.size()) return fail(const_cast<icc_handle*>(h), ICC_ERR_INVALID_ARGUMENT, "n_views differs from the last rolling-shutter camera calibration");
  std::copy(h->camcal_vel.begin(), h->camcal_vel.end(), w_u);
  if (n_without_neighbours) *n_without_neighbours = h->camcal_n_static;
  return ICC_OK;
}

// ---- upstream: static IMU biases (icc_sew.cu) ---------------------------------------------------------------------------------------
icc_status icc_estimate_imu_biases(icc_handle* h, int n, const double* acc, const double* gyr, double gravity_const, double accl_bias[3], double gyro_bias[3]) {
  if (!h || n <= 0 || !acc || !gyr || !accl_bias || !gyro_bias) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  return drive(h, [&](std::string& err) { return imu_biases(h->stream, h->sm_count, n, acc, gyr, gravity_const, accl_bias, gyro_bias, err); });
}

// ---- upstream: static multi-pose IMU intrinsics (icc_static_imu.cu) ---------------------------------------------------------------
void icc_default_static_imu_options(icc_static_imu_options* o) { if (o) default_static_imu_options(o); }

icc_status icc_static_imu_calibration(icc_handle* h, int n, const double* t, const double* acc, const double* gyr, const icc_static_imu_options* opt,
                                      double acc_params[9], double gyr_params[9], double gyr_bias[3], icc_static_imu_summary* summary) {
  if (!h || n < 3 || !t || !acc || !gyr || !acc_params || !gyr_params || !gyr_bias) return ICC_ERR_INVALID_ARGUMENT;   // InitialInterval needs 3 samples
  NEED_DEVICE();
  icc_static_imu_options o; default_static_imu_options(&o);
  if (opt) o = *opt;
  icc_static_imu_summary S;
  const icc_status rc = drive(h, [&](std::string& err) { return static_imu_calibrate(h->stream, n, t, acc, gyr, o, acc_params, gyr_params, gyr_bias, S, h->static_imu_intervals, err); });
  if (rc == ICC_OK && summary) *summary = S;
  return rc;
}

icc_status icc_get_static_imu_intervals(const icc_handle* h, int32_t* buf, int32_t* len) {
  if (!h || !len) return ICC_ERR_INVALID_ARGUMENT;
  const int32_t need = (int32_t)h->static_imu_intervals.size();
  if (!buf) { *len = need; return ICC_OK; }
  if (*len < need) return ICC_ERR_INVALID_ARGUMENT;
  std::copy(h->static_imu_intervals.begin(), h->static_imu_intervals.end(), buf);
  *len = need;
  return ICC_OK;
}

// ---- upstream: Allan variance noise characterisation (icc_allan.cu) -----------------------------------------------------------------
void icc_default_allan_options(icc_allan_options* o) { if (o) default_allan_options(o); }

icc_status icc_allan_variance(icc_handle* h, int n, const double* t, const double* acc, const double* gyr, const icc_allan_options* opt, double params[30], icc_allan_noise noise[6], icc_allan_summary summary[6]) {
  if (!h || !t || !acc || !gyr || !params || !noise || !summary) return ICC_ERR_INVALID_ARGUMENT;
  icc_allan_options o; default_allan_options(&o);
  if (opt) o = *opt;
  if (n < 3 || o.n_clusters < 2) return fail(h, ICC_ERR_INVALID_ARGUMENT, "icc_allan_variance needs n >= 3 samples and n_clusters >= 2");
  NEED_DEVICE();
  const icc_status rc = drive(h, [&](std::string& err) { h->allan_curves = allan::Curves();
    return allan_variance(h->stream, n, t, acc, gyr, o, params, noise, summary, h->allan_curves, err); });
  if (rc != ICC_OK) h->allan_curves = allan::Curves();
  return rc;
}

icc_status icc_get_allan_curves(const icc_handle* h, int channel, int32_t* factors, double* tau, double* sigma2, double* fit_deviation, int32_t* len) {
  if (!h || !len || channel < 0 || channel >= 6) return ICC_ERR_INVALID_ARGUMENT;
  const allan::Curves& C = h->allan_curves;
  const int32_t need = (int32_t)C.factors.size();
  if (!factors) { *len = need; return ICC_OK; }
  if (*len < need || !tau || !sigma2 || !fit_deviation) return ICC_ERR_INVALID_ARGUMENT;
  std::copy(C.factors.begin(), C.factors.end(), factors);
  std::copy(C.tau.begin(), C.tau.end(), tau);
  std::copy(C.sigma2[channel].begin(), C.sigma2[channel].end(), sigma2);
  std::copy(C.fit_deviation[channel].begin(), C.fit_deviation[channel].end(), fit_deviation);
  *len = need;
  return ICC_OK;
}

icc_status icc_get_corner_errors(icc_handle* h, int n, double* err) {
  if (!h || (!err && n != 0)) return ICC_ERR_INVALID_ARGUMENT;
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  if (n != h->P.n_corners) return fail(h, ICC_ERR_INVALID_ARGUMENT, "n must be the number of corners in this shard's solve (icc_num_residuals)");
  CU(cudaSetDevice(h->device));
  { icc_status r = corner_error_pass(h); if (r != ICC_OK) return r; }
  if (n > 0) CU(cudaMemcpyAsync(err, h->d_cerr.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return ICC_OK;
}
icc_status icc_reject_outlier_corners(icc_handle* h, double k_sigma, double min_px, icc_outlier_summary* out) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (!(k_sigma > 0.0) || !std::isfinite(k_sigma) || !(min_px >= 0.0) || !std::isfinite(min_px))
    return fail(h, ICC_ERR_INVALID_ARGUMENT, "k_sigma must be positive and finite, min_px non-negative and finite");
  NEED_DEVICE();
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  CU(cudaSetDevice(h->device));
  return reject_outliers(h, k_sigma, min_px, out);
}
icc_status icc_get_corner_status(const icc_handle* hc, int n_input, int32_t* status) {
  icc_handle* h = const_cast<icc_handle*>(hc);
  if (!h || !status) return ICC_ERR_INVALID_ARGUMENT;
  if (!h->initialised) return fail(h, ICC_ERR_STATE, "icc_batch_init_spline must be called first");
  if (n_input < 0 || (size_t)n_input != h->n_corners_assembled) return fail(h, ICC_ERR_INVALID_ARGUMENT, "n_input must be the number of corners given to icc_set_frames");
  std::fill(status, status + n_input, -1);
  for (const auto& r : h->frame_in) std::fill(status + r.first, status + r.second, h->corners_rejected ? 0 : 1);
  if (h->corners_rejected && h->P.n_corners > 0) {
    std::vector<int> src((size_t)h->P.n_corners);
    CU(cudaSetDevice(h->device));
    CU(cudaMemcpyAsync(src.data(), h->d_csrc.p, src.size() * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    for (const int c : src) status[c] = 1;
  }
  return ICC_OK;
}

// ---- upstream: radon checkerboard corners (icc_board.cu) -------------------------------------------------------------------------------
namespace {
icc_status extract_radon(icc_handle* h, const char* name, bool bgr, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, int corners_x,
                         int corners_y, double f, double* uv_out, int32_t* found, icc_board_summary* summary) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  const int64_t row = (bgr ? 3 : 1) * (int64_t)width;
  if (n_frames < 0 || width < 1 || height < 1 || pitch < row || corners_x < 3 || corners_y < 3 || !(f >= 1.0) || !std::isfinite(f) ||
      (n_frames > 0 && (!frames || !uv_out || !found)))
    return fail(h, ICC_ERR_INVALID_ARGUMENT, std::string(name) + " needs corners_x, corners_y >= 3, a finite downsample factor >= 1, pitch >= " +
                                                 (bgr ? "3 width" : "width") + " and non-NULL frames and outputs");
  NEED_DEVICE();
  icc_board_summary S;
  memset(&S, 0, sizeof S);
  if (n_frames == 0) { if (summary) *summary = S; return ICC_OK; }
  cudaPointerAttributes at;
  bool on_device = false;
  if (cudaPointerGetAttributes(&at, frames) == cudaSuccess) on_device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  else cudaGetLastError();
  const icc_status rc = drive(h, [&](std::string& err) { return extract_radon_board(h->stream, n_frames, width, height, pitch, frames, on_device, bgr, corners_x, corners_y, f, uv_out, found, S, err); });
  if (rc == ICC_OK && summary) *summary = S;
  return rc;
}
}  // namespace

icc_status icc_extract_radon_board(icc_handle* h, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, int corners_x, int corners_y,
                                   double f, double* uv_out, int32_t* found, icc_board_summary* summary) {
  return extract_radon(h, "icc_extract_radon_board", false, n_frames, width, height, pitch, frames, corners_x, corners_y, f, uv_out, found, summary);
}
icc_status icc_extract_radon_board_bgr(icc_handle* h, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames_bgr, int corners_x, int corners_y,
                                       double f, double* uv_out, int32_t* found, icc_board_summary* summary) {
  return extract_radon(h, "icc_extract_radon_board_bgr", true, n_frames, width, height, pitch, frames_bgr, corners_x, corners_y, f, uv_out, found, summary);
}

// ---- upstream: Kalibr AprilGrid corners (icc_aprilgrid.cu) ------------------------------------------------------------------------------
icc_status icc_extract_aprilgrid(icc_handle* h, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, int tags_x, int tags_y,
                                 double f, double* uv_out, int32_t* status_out, int32_t* found, icc_aprilgrid_summary* summary) {
  if (!h) return ICC_ERR_INVALID_ARGUMENT;
  if (n_frames < 0 || width < 1 || height < 1 || pitch < width || tags_x < 1 || tags_y < 1 || tags_x > 64 || tags_y > 64 || !(f >= 1.0) || !std::isfinite(f) ||
      (n_frames > 0 && (!frames || !uv_out || !status_out || !found)))
    return fail(h, ICC_ERR_INVALID_ARGUMENT, "icc_extract_aprilgrid needs tags_x, tags_y in 1..64, a finite downsample factor >= 1, pitch >= width "
                                             "and non-NULL frames and outputs");
  NEED_DEVICE();
  icc_aprilgrid_summary S;
  memset(&S, 0, sizeof S);
  if (n_frames == 0) { if (summary) *summary = S; return ICC_OK; }
  cudaPointerAttributes at;
  bool on_device = false;
  if (cudaPointerGetAttributes(&at, frames) == cudaSuccess) on_device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  else cudaGetLastError();
  const icc_status rc = drive(h, [&](std::string& err) {
    return extract_aprilgrid(h->stream, n_frames, width, height, pitch, frames, on_device, tags_x, tags_y, f, uv_out, status_out, found, S, err);
  });
  if (rc == ICC_OK && summary) *summary = S;
  return rc;
}

icc_status icc_host_alloc_pinned(uint64_t bytes, void** p) {
  if (!p) return ICC_ERR_INVALID_ARGUMENT;
  *p = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return ICC_ERR_NO_DEVICE; }
  if (bytes == 0) return ICC_OK;
  if (cudaHostAlloc(p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); *p = nullptr; return ICC_ERR_CUDA; }
  return ICC_OK;
}
icc_status icc_host_free_pinned(void* p) {
  if (p && cudaFreeHost(p) != cudaSuccess) { cudaGetLastError(); return ICC_ERR_CUDA; }
  return ICC_OK;
}

void icc_trim_device_cache(void) { block_cache().trim(); pinned_cache().trim(); }

}  // extern "C"
