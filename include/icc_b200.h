/* icc_b200.h — C-ABI of the H100-native continuous-time IMU-camera calibration solver.
 *
 * Drop-in boundary for the ONE hot path of urbste/OpenImuCameraCalibrator: everything below
 * OpenICC::core::ImuCameraCalibrator (include/OpenCameraCalibrator/core/imu_camera_calibrator.h:29-118)
 * and SplineTrajectoryEstimator<6> (core/spline_trajectory_estimator.h:31-218), i.e. what the reference
 * delegates to Ceres autodiff + sparse Cholesky + Theia camera projections.  The reference has no FFI layer;
 * each entry point cites the C++ member it replaces.  Plain pointers and sizes only, no torch / C++ types.
 * All arithmetic is FP64; all device work is hand-written sm_90a CUDA; there is NO CPU fallback:
 * every compute entry point fails with ICC_ERR_NO_DEVICE when no CUDA device is usable.
 *
 * Threading: one host thread per handle; one handle per GPU; handles are independent.
 * Ownership: caller owns every input array (copied during the call) and every output buffer.
 */
#ifndef ICC_B200_H_
#define ICC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct icc_handle icc_handle;

typedef enum {
  ICC_OK = 0,
  ICC_ERR_INVALID_ARGUMENT = 1,
  ICC_ERR_NO_DEVICE = 2,       /* CUDA device / driver unusable: the product path never falls back to the CPU */
  ICC_ERR_CUDA = 3,
  ICC_ERR_STATE = 4,           /* call order violated (e.g. optimize before batch_init_spline) */
  ICC_ERR_UNSUPPORTED = 5,     /* outside the solver's limits (e.g. POINTS with more than ~133 board points: border too wide), never a silent fallback */
  ICC_ERR_NUMERIC = 6          /* factorisation broke down / non-finite cost */
} icc_status;

/* theia::CameraIntrinsicsModelType numeric values (pyTheiaSfM@69c3d37); JSON `intrinsic_type` strings are the
 * upper-case names (src/io/read_camera_calibration.cc:59-116).  Intrinsic vectors use Theia's index order:
 *   PINHOLE                   [f, ar, skew, cx, cy, k1, k2]
 *   PINHOLE_RADIAL_TANGENTIAL [f, ar, skew, cx, cy, k1, k2, k3, t1, t2]
 *   FISHEYE                   [f, ar, skew, cx, cy, k1, k2, k3, k4]
 *   FOV                       [f, ar, cx, cy, omega]          (extension: the reference never dispatches FOV)
 *   DIVISION_UNDISTORTION     [f, ar, cx, cy, k]
 *   DOUBLE_SPHERE             [f, ar, skew, cx, cy, xi, alpha]
 *   EXTENDED_UNIFIED          [f, ar, skew, cx, cy, alpha, beta]
 *   OMNI_RADIAL_TANGENTIAL    [f, ar, skew, cx, cy, xi, k1, k2, t1, t2]   (extension, no Theia counterpart: Kalibr's omni-radtan;
 *                             n = z + xi |p|, (mx, my) = (x, y) / n radial-tangentially distorted, then the skewed affine; valid iff
 *                             z > -w |p|, w = xi <= 1 ? xi : 1 / xi)
 *   SCARAMUZZA                [a0, c, e, cx, cy, a2, a3, a4, d]   (extension, no Theia counterpart: Scaramuzza's omnidirectional model as
 *                             OCamCalib calibrates it; the pixel's sensor point (u', v') = A^-1 (u - cx, v - cy), A = [[1, e], [d, c]], sees the ray
 *                             (u', v', a0 + a2 rho^2 + a3 rho^3 + a4 rho^4), rho = |(u', v')|; a point projects through the root of that quartic,
 *                             valid iff z / |(x, y)| > F(rho_max) / rho_max, rho_max = the first stationary point of F(rho) / rho)
 *   PINHOLE_RATIONAL          [f, ar, skew, cx, cy, k1, k2, k3, t1, t2, k4, k5, k6]   (extension, no Theia counterpart: OpenCV's rational
 *                             polynomial model, CALIB_RATIONAL_MODEL, with t1, t2 = OpenCV's p1, p2; (xn, yn) = (x, y) / z, s = xn^2 + yn^2,
 *                             R = (1 + k1 s + k2 s^2 + k3 s^3) / (1 + k4 s + k5 s^2 + k6 s^3), dx = xn R + 2 t1 xn yn + t2 (s + 2 xn^2),
 *                             dy = yn R + t1 (s + 2 yn^2) + 2 t2 xn yn, then the skewed affine; valid iff z > 0 and s < s_max, the first
 *                             s > 0 at which r R(r^2) stops increasing (a root of d(r R)/dr or a pole of R), +inf when there is none)
 *   FISHEYE_RADIAL_TANGENTIAL [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2]   (extension, no Theia counterpart: Kannala-Brandt with
 *                             six radial and two tangential terms, Fisheye62; theta = atan2(|(x, y)|, z), theta_d = theta (1 + k1 theta^2 + ...
 *                             + k6 theta^12), (xr, yr) = (theta_d / |(x, y)|) (x, y), s = xr^2 + yr^2, dx = xr + 2 t1 xr yr + t2 (s + 2 xr^2),
 *                             dy = yr + t1 (s + 2 yr^2) + 2 t2 xr yr, then the skewed affine; t1, t2 as PINHOLE_RADIAL_TANGENTIAL's (OpenCV's p1,
 *                             p2); k1..k4 sit where FISHEYE keeps them; valid iff z > 0 and d theta_d / d theta has no root in (0, theta])
 * ICC_MAX_INTRINSICS is the longest of these vectors. */
#define ICC_MAX_INTRINSICS 13
typedef enum {
  ICC_CAM_PINHOLE = 0,
  ICC_CAM_PINHOLE_RADIAL_TANGENTIAL = 1,
  ICC_CAM_FISHEYE = 2,
  ICC_CAM_FOV = 3,
  ICC_CAM_DIVISION_UNDISTORTION = 4,
  ICC_CAM_DOUBLE_SPHERE = 5,
  ICC_CAM_EXTENDED_UNIFIED = 6,
  ICC_CAM_OMNI_RADIAL_TANGENTIAL = 7,
  ICC_CAM_SCARAMUZZA = 8,
  ICC_CAM_PINHOLE_RATIONAL = 9,
  ICC_CAM_FISHEYE_RADIAL_TANGENTIAL = 10
} icc_camera_model;

/* OpenICC::core::SplineOptimFlags (core/spline_trajectory_estimator.h:17-27), same numeric values. */
enum {
  ICC_FLAG_POINTS = 1 << 0,           /* board points as parameter blocks, HomogeneousVectorParameterization(4) (impl.h:136-152): 3 tangent columns per point,
                                         last in the canonical order; read the result with icc_get_board_points */
  ICC_FLAG_T_I_C = 1 << 1,
  ICC_FLAG_IMU_BIASES = 1 << 2,
  ICC_FLAG_IMU_INTRINSICS = 1 << 3,
  ICC_FLAG_GRAVITY_DIR = 1 << 4,
  ICC_FLAG_CAM_LINE_DELAY = 1 << 5,
  ICC_FLAG_SPLINE = 1 << 6,
  ICC_FLAG_ACC_BIAS = 1 << 7,
  ICC_FLAG_GYR_BIAS = 1 << 8,
  /* Extensions named by the north-star; the reference keeps both quantities fixed (SURVEY.md "Read this first" #3), so with
   * these bits clear they are pass-through exactly like there. */
  ICC_FLAG_CAM_INTRINSICS = 1 << 9,   /* camera intrinsics (Theia parameter vector of the active model) as a parameter block */
  ICC_FLAG_TIME_OFFSET = 1 << 10      /* increment [s] of the IMU->camera time offset applied to every IMU sample time */
};

/* Arguments of ImuCameraCalibrator::BatchInitSpline (src/core/imu_camera_calibrator.cc:21-124). */
typedef struct {
  double T_i_c_init[7];        /* Sophus SE3 storage: quaternion x,y,z,w then translation (impl.h:519,579) */
  double dt_so3_s, dt_r3_s;    /* SplineWeightingData::dt_so3 / dt_r3 (seconds) */
  double std_so3, std_r3;      /* weights are 1/std (imu_camera_calibrator.cc:111,117) */
  double time_offset_imu_to_cam_s;
  double init_line_delay_s;    /* 0 => global shutter path (vision zero-weighted, SURVEY quirk q3) */
  double acc_intrinsics[6];    /* [misYZ, misZY, misZX, sX, sY, sZ]                         (impl.h:1236-1239) */
  double gyr_intrinsics[9];    /* [misYZ, misZY, misZX, misXZ, misXY, misYX, sX, sY, sZ]    (impl.h:1241-1245) */
  double acc_bias[3], gyr_bias[3];
  int32_t dispatch_fov;        /* 0 = reference behaviour (FOV fails -> 1e10 residuals); 1 = enable FOV extension */
  int32_t reserved;
} icc_init_params;

/* Solver knobs: ceres::Solver::Options as set in SplineTrajectoryEstimator::Optimize (impl.h:254-266)
 * plus the Ceres 2.1 defaults that shape the Levenberg-Marquardt path. */
typedef struct {
  double function_tolerance;        /* 1e-4  (impl.h:262) */
  double parameter_tolerance;       /* 1e-7  (impl.h:263) */
  double gradient_tolerance;        /* 1e-10 (Ceres default) */
  double initial_trust_region_radius; /* 1e4 */
  double max_trust_region_radius;   /* 1e16 */
  double min_trust_region_radius;   /* 1e-32 */
  double min_relative_decrease;     /* 1e-3 */
  double min_lm_diagonal;           /* 1e-6 */
  double max_lm_diagonal;           /* 1e32 */
  int32_t jacobi_scaling;           /* 1 */
  int32_t max_consecutive_invalid_steps; /* 5 */
} icc_solver_options;

typedef struct {
  int32_t iterations;               /* LM iterations executed (successful + unsuccessful) */
  int32_t successful_steps;
  int32_t termination;              /* 0 = max iterations, 1 = function tol, 2 = parameter tol, 3 = gradient tol, 4 = failure */
  int32_t num_residuals;            /* scalar residuals per evaluation */
  int32_t num_tangent;              /* active tangent parameters */
  int32_t jacobian_evaluations;
  int32_t cost_evaluations;
  int32_t gpu_launches;             /* CUDA kernels launched inside this optimize call */
  double initial_cost, final_cost;
  double mean_reproj_error;         /* GetMeanReprojectionError (impl.h:993-1072) — return value of Optimize */
  double seconds_total;             /* host wall clock of the optimize call */
  double seconds_jacobian;          /* device time in residual+Jacobian+normal-equation kernels (CUDA events) */
  double seconds_linear_solve;      /* device time in the banded/bordered Cholesky + step kernels */
} icc_summary;

/* Optional cross-rank reduction hook for residual sharding (SURVEY §8(e)): called on the host with the DEVICE pointer
 * of the packed FP64 normal-equation buffer {band, border coupling, border block, gradient, cost}; must sum it in place
 * across ranks (e.g. torch.distributed / ncclAllReduce on the handle's stream) before returning. */
typedef void (*icc_allreduce_fn)(void* device_ptr, int64_t n_doubles, void* cuda_stream, void* user);

/* ---- lifetime --------------------------------------------------------------------------------------------- */
icc_status icc_create(icc_handle** out, int device_ordinal);
void icc_destroy(icc_handle* h);
const char* icc_last_error(const icc_handle* h);          /* never NULL */
const char* icc_version(void);
void icc_default_solver_options(icc_solver_options* o);
icc_status icc_set_solver_options(icc_handle* h, const icc_solver_options* o);

/* ---- problem data (what main() hands to ImuCameraCalibrator, continuous_time_imu_to_camera_calibration.cc:104-199) */
/* theia::Camera intrinsics read at ceres_calib_split_residuals.h:333-336 */
icc_status icc_set_camera(icc_handle* h, int model, const double* intrinsics, int n_intrinsics, int image_width, int image_height);
/* theia::Track::Point() homogeneous board points, id = index (app :111-119).  After icc_batch_init_spline only the coordinates may change
 * (same count); the new points reach the device state at once. */
icc_status icc_set_board_points(icc_handle* h, int n_points, const double* xyzw);
/* Views of the calibration dataset (app :131-161): timestamp [s], observed corners (CSR over frames), and the per-view
 * pose prior used by BatchInitSO3R3VisPoses: q_wc (x,y,z,w) = R_cw^T and camera position p_wc (impl.h:290-300). */
icc_status icc_set_frames(icc_handle* h, int n_frames, const double* timestamps_s, const int32_t* corner_offsets /* n_frames+1 */,
                          const int32_t* point_ids, const double* uv, const double* q_wc_xyzw, const double* p_wc);
/* CameraTelemetryData accelerometer/gyroscope streams (src/io/read_telemetry.cc:49-56) */
icc_status icc_set_imu(icc_handle* h, int n_samples, const double* timestamps_s, const double* accel_xyz, const double* gyro_xyz);

/* ---- ImuCameraCalibrator API -------------------------------------------------------------------------------- */
/* BatchInitSpline (imu_camera_calibrator.cc:21-124): spline time range, knot counts, knot initialisation, bias
 * splines, measurement wiring (CalcTimes impl.h:763-788), gravity initialisation; uploads everything to HBM. */
icc_status icc_batch_init_spline(icc_handle* h, const icc_init_params* p);
/* ---- bias splines (extension: the reference fixes InitBiasSplines(bias, bias, 10 s, 10 s, 1.0, 0.1), imu_camera_calibrator.cc:79-85) ----
 * icc_set_bias_splines: knot spacing [s] of the accelerometer / gyroscope bias splines; a value <= 0 selects the reference's 10 s, and so does
 * never calling it.  Knot counts stay duration / dt + 3.  icc_set_bias_random_walk: random-walk densities per axis in SI units, Kalibr's
 * accelerometer_random_walk [m/s^3/sqrt(Hz)] and gyroscope_random_walk [rad/s^2/sqrt(Hz)]; NULL turns that sensor's prior off (the default).
 * Both are read by the next icc_batch_init_spline.  A sensor with densities adds, per bias-spline segment s = 0 .. n-3, Gauss-Legendre node
 * g = 0, 1 (u_g = 1/2 -+ 1/(2 sqrt 3)) and axis a, the residual r = sqrt(dt / 2) b'_a(u_g) / q_a, so that 1/2 sum r^2 is the Wiener-process
 * negative log-likelihood 1/2 int |b'|^2 / q^2 dt of the whole spline.  The rows are part of the problem under every flag set (their cost
 * always counts); they have columns where ACC_BIAS / GYR_BIAS / IMU_BIASES free the knots.  Residual order of icc_evaluate: [vision | accel |
 * gyro | acc-bias prior | gyr-bias prior], segment-major, then node, then axis.  Under sharding only shard 0 holds the rows.  The bias box
 * (|b| <= 1.0 / 0.1) is unchanged.  Free bias knots are border columns of the solver: too many give ICC_ERR_UNSUPPORTED from the solve.
 * Non-finite, zero or negative densities, or a spacing that is not finite or outside [1 ns, 1e9 s]: ICC_ERR_INVALID_ARGUMENT.  Host state only. */
icc_status icc_set_bias_splines(icc_handle* h, double acc_dt_s, double gyr_dt_s);
icc_status icc_set_bias_random_walk(icc_handle* h, const double acc_q[3] /* nullable */, const double gyr_q[3] /* nullable */);
/* prior rows of this shard's problem (0 without densities, and on shards other than 0) */
icc_status icc_num_bias_prior_residuals(const icc_handle* h, int* n);
/* SetKnownGravityDir (imu_camera_calibrator.cc:126-128) */
icc_status icc_set_known_gravity_dir(icc_handle* h, const double g[3]);
/* Residual sharding: keep only frames/IMU samples in shard `rank` of `world` (time-sliced, equal residual counts);
 * knots stay replicated.  Must be called before icc_batch_init_spline.  world = 1 restores the full problem. */
icc_status icc_set_shard(icc_handle* h, int rank, int world);
icc_status icc_set_allreduce(icc_handle* h, icc_allreduce_fn fn, void* user);
/* Native multi-GPU path: an NCCL communicator owned by the library (bound to the process' NCCL with dlopen).  One rank creates the
 * id, every rank creates its communicator (collective call), the handle borrows it: icc_set_comm sets the residual shard to the
 * communicator's (rank, world) and routes every cross-rank sum through ncclAllReduce on the solver's stream -- one all-reduce of the
 * packed normal equations per Jacobian evaluation, one 8-byte all-reduce per candidate cost.  One process per GPU (the drop-in
 * CLI's --gpus mode spawns one rank process per device).  Reference: SURVEY.md §8(e). */
#define ICC_COMM_ID_BYTES 128
typedef struct icc_comm icc_comm;
icc_status icc_comm_unique_id(unsigned char id[ICC_COMM_ID_BYTES]);
icc_status icc_comm_create(icc_comm** out, const unsigned char id[ICC_COMM_ID_BYTES], int rank, int world, int device_ordinal);
void icc_comm_destroy(icc_comm* c);
int icc_comm_rank(const icc_comm* c);
int icc_comm_world(const icc_comm* c);
int icc_comm_nccl_version(void);              /* 0 when NCCL could not be bound */
const char* icc_comm_last_error(void);        /* never NULL; thread local */
icc_status icc_set_comm(icc_handle* h, icc_comm* c);   /* NULL detaches (single-GPU, shard 0 of 1) */
/* Optimize (imu_camera_calibrator.cc:163-168 -> impl.h:254-276): LM over the blocks selected by `flags`. */
icc_status icc_optimize(icc_handle* h, int max_iterations, int flags, icc_summary* summary);

/* ---- getters (imu_camera_calibrator.h:48-77; impl.h:898-1072,1180-1234) -------------------------------------- */
icc_status icc_get_T_i_c(const icc_handle* h, double T_i_c[7]);
icc_status icc_get_gravity(const icc_handle* h, double g[3]);
icc_status icc_get_line_delay(const icc_handle* h, double* line_delay_s);
/* extension outputs: current camera intrinsics (n = model's parameter count) and time_offset_imu_to_cam_s (input + estimated increment) */
icc_status icc_get_camera_intrinsics(const icc_handle* h, double* intrinsics, int n);
icc_status icc_get_time_offset(const icc_handle* h, double* time_offset_s);
icc_status icc_get_num_knots(const icc_handle* h, int* n_so3, int* n_r3, int* n_acc_bias, int* n_gyr_bias);
icc_status icc_get_knots(const icc_handle* h, double* so3_xyzw, double* r3_xyz, double* acc_bias_xyz, double* gyr_bias_xyz); /* any may be NULL */
icc_status icc_set_knots(icc_handle* h, const double* so3_xyzw, const double* r3_xyz, const double* acc_bias_xyz, const double* gyr_bias_xyz);
icc_status icc_set_T_i_c(icc_handle* h, const double T_i_c[7]);
icc_status icc_set_line_delay(icc_handle* h, double line_delay_s);
icc_status icc_get_mean_reprojection_error(icc_handle* h, double* err);

/* ---- outlier corners between spline solves (extension: the reference has no per-corner rejection) -----------------------------------
 * The error of a corner is e = sqrt(rx^2 + ry^2) of its unweighted residual pair at the current state with rolling-shutter timing: in the
 * pixel mode exactly the terms icc_get_mean_reprojection_error averages, with ICC_REPROJ_ERROR_TANGENT the scaled tangent residual the solve
 * minimises.  A pair with rx == 0 || ry == 0 (the reference's quirk in GetMeanReprojectionError, impl.h:1058-1064) is neither counted nor
 * rejected; a failed projection (the constant 1e10 pair) is not counted and always rejected.
 * icc_reject_outlier_corners sums e^2 and the count of the counted corners over the shards (the cross-rank sum of the solve), so every rank
 * uses the same threshold = max(min_px, k_sigma * rms_px), and removes from this shard's solve every corner with e > threshold.  The state,
 * the solver options and the inputs of icc_set_frames are not changed; icc_num_residuals, icc_evaluate, icc_get_eval_schedule and the next
 * icc_optimize see the reduced set until icc_batch_init_spline assembles the problem again.  A frame left without corners keeps its knots
 * (the IMU holds them).  ICC_ERR_STATE before icc_batch_init_spline; k_sigma <= 0 or non-finite, min_px negative or non-finite:
 * ICC_ERR_INVALID_ARGUMENT. */
typedef struct {
  int64_t n_corners;        /* corners in the solve before this call (all shards) */
  int64_t n_rejected;       /* removed by this call (all shards), failed projections included */
  int64_t n_failed;         /* of those: corners whose projection failed (the 1e10 residuals) */
  int32_t n_frames_emptied; /* frames left without corners (they leave the vision schedule; their knots stay, held by the IMU) */
  int32_t reserved;
  double rms_px;            /* sqrt(mean e^2) over the counted corners (all shards) */
  double threshold_px;      /* max(min_px, k_sigma * rms_px) */
} icc_outlier_summary;
/* e of every corner in this shard's solve, in frame order; n = that count (icc_num_residuals' n_vision / 2 on the rolling-shutter path) */
icc_status icc_get_corner_errors(icc_handle* h, int n, double* err_px);
icc_status icc_reject_outlier_corners(icc_handle* h, double k_sigma, double min_px, icc_outlier_summary* out /* nullable */);
/* per corner given to icc_set_frames (n_input = their count): 1 in this shard's solve, 0 rejected, -1 not assembled here (other shard,
 * frame outside the spline).  Host only. */
icc_status icc_get_corner_status(const icc_handle* h, int n_input, int32_t* status);
/* number of IMU samples kept by BatchInitSpline and their (offset-corrected) timestamps / raw readings (app :265-327) */
icc_status icc_get_num_imu_used(const icc_handle* h, int* n);
icc_status icc_get_imu_used(const icc_handle* h, double* t_s, double* accel_xyz, double* gyro_xyz);
/* Knot-interval cells of the kept IMU samples (inspection / tests): maximal runs [i_begin, i_end) of kept samples that lie in the same
 * knot interval of all four splines, i.e. share CalcTimes' segment indices (impl.h:763-788); 6 int32 per cell:
 * s_so3, s_r3, s_acc_bias, s_gyr_bias, i_begin, i_end.  The evaluation kernels stage one knot window per cell. */
icc_status icc_get_num_imu_cells(const icc_handle* h, int* n);
icc_status icc_get_imu_cells(const icc_handle* h, int32_t* cells6);
/* Schedule of the persistent Jacobian kernel (inspection / tests).  The corners of the non-empty frames and the samples of the IMU
 * cells form two packed streams, each unit padded to a multiple of 4 positions; each stream is walked in chunks of up to 32
 * positions from at most two consecutive units and cut into even per-warp runs.  counts4 = {vision chunks, IMU chunks, vision
 * runs, IMU runs}; vitems3 / iitems3 (3 int32 per run, either may be NULL): first unit (index among the non-empty frames / cells),
 * first stream position, end stream position.  ICC_ERR_STATE before icc_batch_init_spline.  The environment variable
 * ICC_TMEM_RUNS=n, read by icc_batch_init_spline, caps the runs per stream at n (tests).  Host only: also works on a host-only
 * (device -1) handle, whose run count assumes the 132 SMs of an H100 SXM. */
icc_status icc_get_eval_schedule(const icc_handle* h, int32_t counts4[4], int32_t* vitems3, int32_t* iitems3);
/* GetAngularVelocity / GetAcceleration / GetGyroBias / GetAcclBias / GetPose evaluated on the GPU for n timestamps [ns];
 * valid[i] = 0 where CalcTimes rejects the timestamp (outputs left untouched there). Any output may be NULL. */
icc_status icc_eval_trajectory(icc_handle* h, int n, const int64_t* t_ns, double* gyro_xyz, double* accel_xyz,
                               double* gyro_bias_xyz, double* accel_bias_xyz, double* pose_q_xyzw, double* pose_p, int32_t* valid);

/* ---- test / measurement surface ----------------------------------------------------------------------------- */
icc_status icc_num_residuals(const icc_handle* h, int* n_vision, int* n_accel, int* n_gyro);   /* scalar residual counts */
icc_status icc_num_tangent(const icc_handle* h, int flags, int* n);
/* One evaluation at the current state.  Canonical tangent order: so3 knots (3 each), r3 knots (3 each), T_i_c (6: upsilon,
 * omega), gravity (3), line delay (1), acc-bias knots (3 each), gyr-bias knots (3 each), accelerometer intrinsics (6),
 * gyroscope intrinsics (9), camera intrinsics (model count), time-offset increment (1) — only blocks active under `flags`.
 * residuals: [vision 2/corner in frame order | accel 3/sample | gyro 3/sample | bias random-walk prior rows (icc_set_bias_random_walk)].  hessian_dense: n x n row-major J^T J
 * (small problems only).  Any output may be NULL. */
icc_status icc_evaluate(icc_handle* h, int flags, double* cost, double* residuals, double* gradient, double* hessian_dense);
/* Run exactly `n` LM iterations (no convergence test) from the current state; used by bench.py as the timed "step". */
/* J^T J V for nvec caller vectors (canonical tangent order, one vector after the other) from the packed normal equations of the
 * current state: full-size parity of the reduced system without a dense Hessian (evaluation helper, like icc_evaluate). */
icc_status icc_normal_matvec(icc_handle* h, int flags, int nvec, const double* V, double* HV);
/* Elimination plan of the damped normal-equation solve (nested dissection of the knot band, see DESIGN.md §3.2).
 * Level 0 cuts the nk knot columns into P chunks: chunk c owns len + (c < rem) interior columns, P - 1 separators of kd columns
 * lie between them.  S[l] (l = 1..L+1) is the separator-block count of reduced system l; levels 1..L eliminate every other block. */
typedef struct icc_solver_plan_info {
  int32_t valid;               /* 0: no plan fits the shared-memory limits (the solve returns ICC_ERR_UNSUPPORTED) */
  int32_t nk, kd, nb;          /* knot (band) columns, half bandwidth, border columns */
  int32_t P, len, rem, L;
  int32_t cl_global, cs_global;  /* level-0 local border block / root border block live in HBM instead of shared memory */
  int32_t stage0;              /* level-0 back-substitution may stage its El rows in shared memory */
  int32_t WS_A;                /* level-0 window slots (power of two) */
  int32_t backsub0_staged;     /* level-0 chunks whose back-substitution is staged (interior <= 128 columns and stage0) */
  int32_t max_leaf;            /* len + (rem > 0) */
  int32_t S[16];
  int64_t smem_bytes[5];       /* dynamic shared memory: eliminate, reduce, root, level-0 back-substitution, level >= 1 back-substitution */
  int64_t workspace_doubles;   /* device workspace of the plan (0 when not valid) */
} icc_solver_plan_info;
/* The plan icc_solve_normal_equations would use under `flags` with `chunks` level-0 chunks (0 = the planner's choice).  Host
 * only: also works on a host-only (device -1) handle. */
icc_status icc_solver_plan(icc_handle* h, int flags, int chunks, icc_solver_plan_info* plan);
/* One damped solve of the normal equations that the preceding icc_evaluate (with gradient or Hessian) or icc_normal_matvec left
 * in the handle for the same `flags`; no evaluation, the state is not touched (ICC_ERR_STATE when those normal equations are not
 * current).  Jacobi scale s = 1/(1+sqrt(H_ii)) (1 without jacobi_scaling), then (S H S + D) y = -S g with
 * D = clamp(H_ii s_i^2, min_lm_diagonal, max_lm_diagonal) / radius, delta = S y: exactly the step of one LM iteration at that
 * radius.  `chunks` as in icc_solver_plan; a plan that does not fit returns ICC_ERR_UNSUPPORTED before any launch.
 * Outputs (canonical tangent order, any may be NULL): delta, scale, h_diag (diag(H) as the solver read it), the model cost change
 * -(g^T delta + delta^T H delta / 2), step_ok (0 when a pivot was not positive: the delta output is then not written), plan. */
icc_status icc_solve_normal_equations(icc_handle* h, int flags, double radius, int chunks, double* delta, double* scale, double* h_diag,
                                      double* model_change, int32_t* step_ok, icc_solver_plan_info* plan);
icc_status icc_lm_iterations(icc_handle* h, int n, int flags, icc_summary* summary);
/* CUDA kernels this library has launched in this process, all handles together (tests: a refused call launches nothing). */
int64_t icc_kernel_launch_count(void);
/* Run `n` bare residual+Jacobian+normal-equation evaluations (the residual-eval kernels only); device ms per evaluation. */
icc_status icc_time_evaluations(icc_handle* h, int n, int flags, int with_jacobian, double* ms_per_eval);
/* The handle's cudaStream_t (so that callers can bracket calls with their own CUDA events on the launching stream). */
void* icc_get_stream(icc_handle* h);

/* ---- upstream row f1 (SURVEY.md §8(f)): per-view board poses, i.e. what fills the pose dataset the hot CLI reads -----------
 * PoseEstimator::EstimatePosesFromJson (src/core/pose_estimator.cc:92-191): every corner is undistorted to the normalised image
 * plane (theia::Camera::PixelToNormalizedCoordinates, :129-130), a calibrated absolute pose is estimated (RANSAC PnP,
 * :54-66; squared normalised reprojection error threshold 0.004 * image_height / image_diagonal, :100-101; >= 6 inliers, :65),
 * then refined on the inliers by theia::BundleAdjustView with a Huber(1.345) loss (:44-48, :86-87); views with fewer than
 * `min_points` corners (pose_estimator.h:72, default 8) or a mean reprojection error above `max_reproj_error` (:181) are dropped.
 * Here: camera + board points must have been set (icc_set_camera / icc_set_board_points; the board must be planar up to a few per cent of its size -- the
 * homography only starts the refinement, which uses the real 3-D points);
 * one warp per view computes a normalised homography initialisation and the Levenberg-Marquardt refinement on the same cost,
 * so that the converged pose is the reference's BundleAdjustView optimum (RANSAC's random minimal samples are not reproduced:
 * the inlier set is taken with the same threshold around the refined pose).
 * Outputs (per view, caller-owned): q_wc (x,y,z,w) = R_cw^T and p_wc exactly as icc_set_frames consumes them, the mean
 * normalised reprojection error, valid (1 / 0).  max_reproj_error <= 0 selects 0.004 * image_height; min_points <= 0 selects 8.
 * Wide-angle lenses: the normalised plane cannot hold a ray 90 degrees or more off the axis, so such corners are lost (and views with them);
 * icc_set_pose_error(h, ICC_POSE_ERROR_TANGENT) switches this call and icc_optimize_board_points to unit bearings (icc_pixels_to_bearings)
 * and the local tangent reprojection error.  Then mean_reproj_error, the inlier threshold and max_reproj_error are in tangent units. */
icc_status icc_estimate_board_poses(icc_handle* h, int n_frames, const int32_t* corner_offsets /* n_frames+1 */, const int32_t* point_ids,
                                    const double* uv, double max_reproj_error, int min_points,
                                    double* q_wc_xyzw, double* p_wc, double* mean_reproj_error, int32_t* valid);
/* PoseEstimator::FilterBadPoses (src/core/pose_estimator.cc:238-261), the last step of estimate_camera_poses_from_checkerboard
 * (app :66-67): views whose camera height p_wc.z differs from the median height of the valid views by more than |median| are dropped
 * (poses far away or on the wrong side of the board).  Host logic only: valid[] is updated in place; h may be NULL. */
icc_status icc_filter_bad_poses(icc_handle* h, int n_views, const double* p_wc, int32_t* valid);
/* --optimize_board_points of the pose app (app :61-65): PoseEstimator::OptimizeBoardPoints (pose_estimator.cc:193-224) =
 * theia::BundleAdjustTracks over the board points seen in more than `min_observations` (<= 0 selects min_num_obs_for_optim_ = 30,
 * pose_estimator.h:78) inlier observations, every camera constant, residual = normalised pinhole reprojection error of the
 * undistorted corners, Huber(1.345); then PoseEstimator::OptimizeAllPoses (:226-236) = BundleAdjustView of every valid view on the
 * new points.  q_wc / p_wc / valid are in-out (as returned by icc_estimate_board_poses); the handle's board points are replaced
 * (also returned in board_xyzw_out, w = 1 for optimised points).  With cameras fixed every point is an independent 3-parameter
 * problem: one warp per point on the GPU.  The empirical covariances the reference prints (:212-223) are not computed. */
icc_status icc_optimize_board_points(icc_handle* h, int n_frames, const int32_t* corner_offsets, const int32_t* point_ids, const double* uv,
                                     double max_reproj_error, int min_points, int min_observations,
                                     double* q_wc_xyzw, double* p_wc, double* mean_reproj_error /* nullable */, int32_t* valid,
                                     double* board_xyzw_out /* nullable, 4 per board point */, int32_t* n_points_optimized /* nullable */);
/* current board points of the handle (icc_set_board_points, or refined by icc_optimize_board_points / icc_calibrate_camera / a spline
 * solve with ICC_FLAG_POINTS) */
icc_status icc_get_board_points(const icc_handle* h, double* xyzw, int n);
/* theia::Camera::PixelToNormalizedCoordinates / z for `n` pixels with the handle's camera: xy_out[2n], ok[n] (nullable). */
icc_status icc_pixels_to_normalized(icc_handle* h, int n, const double* uv, double* xy_out, int32_t* ok);
/* Unit bearing vectors of `n` pixels with the handle's camera: xyz_out[3n], ok[n] (nullable; 0 where the ray reprojects more than 1e-6 px
 * away).  Pinhole, PinholeRadialTangential, FOV and DivisionUndistortion give icc_pixels_to_normalized's ray normalised; Fisheye's ray
 * stays in z > 0 (the model maps p and -p to one pixel); DoubleSphere, ExtendedUnified and OmniRadialTangential reach their whole domain,
 * z <= 0 included; Scaramuzza back-projects in closed form (ok = 0 beyond rho_max); PinholeRational gives icc_pixels_to_normalized's
 * ray normalised, ok = 0 where it would land outside the model's domain. */
icc_status icc_pixels_to_bearings(icc_handle* h, int n, const double* uv, double* xyz_out, int32_t* ok);

/* Residual of the per-view pose refinement, the inlier test and the board-point refinement of icc_estimate_board_poses and
 * icc_optimize_board_points (not of icc_calibrate_camera, which keeps the normalised start).
 *   ICC_POSE_ERROR_NORMALIZED (default): the reference's normalised pinhole error of BundleAdjustView.
 *   ICC_POSE_ERROR_TANGENT: corners are unit bearings b with a tangent basis (e1, e2); a predicted camera-frame point d scores
 *     r = (e1.d, e2.d) / (b.d), with a 1e6 cost where b.d <= 0.  The start rotates a view's bearings so that their mean is the axis and
 *     takes the homography of those within 80 degrees of it; the rules (min_points, >= 6 inliers, the squared-error threshold, the mean
 *     error against max_reproj_error) are kept, on the tangent error.  mean_reproj_error is then in tangent units.
 * Any other mode is ICC_ERR_INVALID_ARGUMENT.  Host state only: also accepted by a host-only handle. */
#define ICC_POSE_ERROR_NORMALIZED 0
#define ICC_POSE_ERROR_TANGENT 1
icc_status icc_set_pose_error(icc_handle* h, int mode);

/* Vision residual of the spline solve (icc_optimize, icc_lm_iterations, icc_evaluate and the other entry points that take flags).
 *   ICC_REPROJ_ERROR_PIXEL (default): the reference's pixel residual project(p_c) - (u, v).
 *   ICC_REPROJ_ERROR_TANGENT: the local tangent reprojection error.  Each corner is its unit bearing b (icc_pixels_to_bearings, formed once
 *     at icc_batch_init_spline with the intrinsics set then) with the tangent basis (e1, e2) of icc_set_pose_error, and the predicted
 *     camera-frame point p_c scores r = s (e1.p_c, e2.p_c) / (b.p_c).  s = sqrt(|det J0|), J0 = d(u, v)/d(x, y) of the camera at the
 *     principal ray, keeps r in pixels at the image centre, the scale the IMU weights assume.  A corner whose bearing cannot be formed is a
 *     zero residual with zero Jacobian rows; b.p_c <= 0 gives the constant 1e10 with zero rows, like a failed projection of the pixel
 *     residual.  No camera model is evaluated during the solve, so a corner only drops out when its prediction is 90 degrees or more off
 *     its own ray.  Any call with ICC_FLAG_CAM_INTRINSICS is ICC_ERR_UNSUPPORTED (the bearings are fixed by the intrinsics) and changes
 *     nothing.  icc_evaluate returns the scaled tangent residuals; summary.mean_reproj_error and icc_get_mean_reprojection_error stay
 *     in pixels in either mode.
 * ICC_ERR_STATE after icc_batch_init_spline; any other mode is ICC_ERR_INVALID_ARGUMENT.  Also accepted by a host-only handle. */
#define ICC_REPROJ_ERROR_PIXEL 0
#define ICC_REPROJ_ERROR_TANGENT 1
icc_status icc_set_reprojection_error(icc_handle* h, int mode);

/* Shutter of icc_estimate_board_poses and icc_optimize_board_points.  line_delay_s = 0 (the default) is the global shutter: one rigid pose per
 * view, and frame_t_s may be NULL.  line_delay_s > 0 is a rolling shutter: pixel row v of a view is exposed v * line_delay_s after its frame
 * time frame_t_s[i] (the rule of the reference's RS functor, feature.y() * line_delay), and the reported pose is the one at the frame time
 * (row 0).  Over one readout the camera moves with constant camera-frame angular velocity w and linear velocity u, so a corner seen at
 * tau = v * line_delay_s is predicted from P(tau) = exp(-tau [w]x) (R_cw X + t_cw - tau u) with either residual of icc_set_pose_error.
 * The velocities are not free unknowns; they come from each view's neighbours in time.  The views are sorted by time; a view's neighbours are
 * the nearest valid views before and after it whose time differs by more than 0 and by at most 2.5 x the median positive spacing of all
 * view times.  With both neighbours p and n:  w = R_wc,f^T R_wc,p Log(R_wc,p^T R_wc,n) / (t_n - t_p),  u = R_wc,f^T (p_wc,n - p_wc,p) / (t_n - t_p);
 * with one, the same between it and the view; with none, w = u = 0 and the view keeps the global-shutter model.
 * icc_estimate_board_poses runs its global-shutter pass, then exactly two rolling-shutter passes.  Each pass computes the velocities from the
 * current poses and refines every valid view from its pose as icc_optimize_board_points does (usable corners, refinement, inlier threshold,
 * refinement, mean error, max_reproj_error); a view dropped by a pass stays dropped.  icc_optimize_board_points runs one such pass on the
 * given poses, refines the board points with the corners at their row times and the velocities of the new poses, and one more pass.
 * The next pose call must pass n_frames views (else ICC_ERR_INVALID_ARGUMENT).  A negative or non-finite delay or time, or n_frames <= 0 /
 * frame_t_s NULL with a positive delay, is ICC_ERR_INVALID_ARGUMENT.  Host state only: also accepted by a host-only handle. */
icc_status icc_set_pose_rolling_shutter(icc_handle* h, double line_delay_s, int32_t n_frames, const double* frame_t_s);
/* The velocities of the last rolling-shutter pose call on this handle: w_u[6 * n_frames] = (w, u) per view at its frame time (zero for a view
 * that was not valid before that call's last pass, or that had no neighbour), n_without_neighbours (nullable) = the number of valid views
 * without a neighbour.  ICC_ERR_STATE before any such call; ICC_ERR_INVALID_ARGUMENT when n_frames differs from that call's. */
icc_status icc_get_pose_velocities(const icc_handle* h, int32_t n_frames, double* w_u, int32_t* n_without_neighbours);

/* ---- upstream row f3 (SURVEY.md §8(f)): IMU-to-camera rotation + time offset initialiser -----------------------------------
 * ImuToCameraRotationEstimator::EstimateCameraImuRotation (src/core/imu_to_camera_rotation_estimator.cc:116-274) together with
 * the preparation done by applications/estimate_imu_to_camera_rotation.cc:96-173: view rotations q_cw (quaternion of
 * theia::Camera::GetOrientationAsRotationMatrix, app :125-127) resampled to the median frame interval, interpolated to the IMU
 * rate, differentiated to a visual angular velocity, both streams smoothed by a 15-tap moving average, then a golden-section
 * search over the time offset in [-1, 1] s (tolerance 1e-4 s) around the closed-form rotation (+ gyroscope bias) fit.
 * Inputs: views (any order; timestamps already include the first-image offset of app :80-86), gyroscope samples (any order);
 * gyro_bias_in = NULL enables the bias estimation (EnableGyroBiasEstimation, app :63-67), otherwise it is subtracted from the
 * samples (app :99-100) and returned unchanged.  Outputs: q_gyro_to_cam (x,y,z,w) as written to "gyro_to_camera_rotation",
 * the time offset "time_offset_gyro_to_cam", the gyroscope bias, the final alignment error and the number of iterations.
 * One documented divergence: where the reference's InterpolateVector3d reads one element past the end of its input
 * (utils.cc:250-256, undefined behaviour) the last sample is used as is. */
icc_status icc_estimate_imu_to_camera_rotation(icc_handle* h, int n_views, const double* view_t_s, const double* q_cw_xyzw,
                                               int n_imu, const double* imu_t_s, const double* gyro_xyz, const double* gyro_bias_in /* 3 or NULL */,
                                               double* q_gyro_to_cam_xyzw /* 4 */, double* time_offset_s, double* gyro_bias_out /* 3 */,
                                               double* alignment_error, int32_t* iterations);

/* ---- upstream row f2 (SURVEY.md §8(f)): spline error weighting -----------------------------------------------------------------
 * python/sew.py:knot_spacing_and_variance (python/sew.py:201-234) as called by python/get_sew_for_dataset.py:38-48 for the
 * accelerometer (q_r3 = 0.96, dt in [0.01, 0.15]) and the gyroscope (q_so3 = 0.98, dt in [0.01, 0.2]): the largest uniform knot
 * spacing whose cubic-B-spline interpolation response keeps `quality` of the signal energy, and the variance of the spline fit
 * error at that spacing (its square root is the "weighting_factor" of spline_error_weighting_json).
 * signal_xyz: n x 3 samples; times_s: their timestamps (mean rate is used); min_dt / max_dt <= 0 select the defaults of sew.py
 * (1 / rate and n / 4 / rate).  spectrum (nullable, n doubles) receives the reference spectrum Xhat (make_reference_spectrum). */
icc_status icc_spline_error_weighting(icc_handle* h, int n, const double* times_s, const double* signal_xyz, double quality, double min_dt, double max_dt,
                                      double* knot_spacing, double* variance, double* spectrum);

/* ---- upstream row f4 (SURVEY.md §8(f)): camera intrinsic calibration ----------------------------------------------------------
 * CameraCalibrator::CalibrateCameraFromJson / RunCalibration (src/core/camera_calibrator.cc:221-389, :131-219) behind
 * applications/calibrate_camera.cc: every view of the corner file gets an initial pose and focal length, views closer than
 * `grid_size` to an already accepted camera position are skipped (:313-325), then theia::BundleAdjustViews runs three times over
 * all view poses + ONE shared intrinsic vector with a Huber(1.345) loss (:140-144):
 *   stage 1  focal length (+ radial distortion unless PINHOLE), poses free (:149-160); views with a mean error > 5 px removed (:162)
 *   stage 2  principal point only, poses constant (:167-174)
 *   stage 3  principal point + focal length + aspect ratio (+ radial for PINHOLE, + tangential for PINHOLE_RADIAL_TANGENTIAL),
 *            poses free (:184-198); views with a mean error > 2 px removed (:200); fewer than 10 views left = failure (:202-205)
 * The residual is theia::ReprojectionError: CameraToPixelCoordinates(intr, R_cw (X - c)) - feature [px].  "Radial distortion" is
 * Theia's per-model subset (k1,k2 | k1..k3 | k1..k4 | k | xi,alpha | alpha,beta | omega).  Initial intrinsics as in AddView
 * (:84-129): principal point = image centre, aspect ratio 1, skew 0, DOUBLE_SPHERE xi = -0.25 alpha = 0.5, EXTENDED_UNIFIED
 * alpha = 0.5 beta = 1, DIVISION_UNDISTORTION k = distortion_init, everything else 0.
 * Initial poses: pass q_wc_init / p_wc_init (+ init_valid) and focal_length_init > 0 to start from your own estimates (what the
 * reference gets from Theia's RANSAC minimal solvers, which are not reproduced), or NULL / <= 0 to have them estimated here:
 * focal length = median over the views of the closed-form estimate from the board homography (Zhang's constraints, principal
 * point at the image centre), poses = homography decomposition + Huber pose refinement under that pinhole camera; for the
 * non-pinhole models focal length, a division-model distortion and the poses are then refined jointly (the quantities
 * utils::initialize_radial_undistortion_camera hands the reference, :283-306) before the target model takes over.
 * Needs icc_set_board_points (planar board for the internal initialiser).
 * Outputs (caller-owned): intrinsics in Theia's order for `model`, max(10, its parameter count) entries (10 for every model but
 * PINHOLE_RATIONAL and FISHEYE_RADIAL_TANGENTIAL, 13 for them; unused entries zero); per view q_wc / p_wc (as icc_set_frames consumes them),
 * the mean reprojection error [px] (GetReprojErrorOfView) and used[v] = 1 for the views that survive to the end.
 * summary->success = 0 (status still ICC_OK) when fewer than min_num_views views remain, like RunCalibration returning false. */
typedef struct icc_camcal_options {
  double grid_size;                  /* SetGridSize (calibrate_camera.cc:33-35); < 0 selects 0.04 m, 0 keeps every view */
  double function_tolerance;         /* <= 0 selects theia's 1e-6 */
  double parameter_tolerance;        /* <= 0 selects theia's 1e-8 */
  double gradient_tolerance;         /* <= 0 selects theia's 1e-10 */
  double huber_width;                /* <= 0 selects 1.345 (camera_calibrator.cc:143) */
  double max_view_error_stage1_px;   /* <= 0 selects 5.0 (:162) */
  double max_view_error_final_px;    /* <= 0 selects 2.0 (:200) */
  int32_t min_num_views;             /* camera_calibrator.h:84; <= 0 selects 10 */
  int32_t max_num_iterations;        /* theia::BundleAdjustmentOptions (external) default 100 per stage; <= 0 selects it */
  int32_t optimize_board_points;     /* --optimize_board_points (camera_calibrator.cc:207-216): BundleAdjustTracks on the board points with
                                        constant cameras, then the full BundleAdjustViews again; read the points with icc_get_board_points */
  int32_t reserved;
} icc_camcal_options;
typedef struct icc_camcal_summary {
  int32_t success;
  int32_t n_views_initialized;       /* views with an initial pose */
  int32_t n_views_selected;          /* ... that also passed the grid filter */
  int32_t n_views_used;              /* ... that survived both removal passes */
  int32_t iterations[3];             /* LM iterations per stage */
  int32_t termination[3];            /* icc_summary.termination codes per stage */
  int32_t gpu_launches;
  int32_t init_iterations;           /* LM iterations of the internal initialiser's joint refinement (0 when poses / focal length are given) */
  int32_t n_points_optimized;        /* board points refined by optimize_board_points */
  int32_t reserved;
  double focal_length_init;
  double initial_cost;               /* cost at the start of stage 1 */
  double final_cost[3];              /* cost at the end of each stage */
  double final_reproj_error;         /* mean over the used views of their mean reprojection error [px] (camera_calibrator.cc:352-366) */
  double seconds_total;
} icc_camcal_summary;
icc_status icc_calibrate_camera(icc_handle* h, int model, int image_width, int image_height,
                                int n_views, const int32_t* corner_offsets /* n_views+1 */, const int32_t* point_ids, const double* uv,
                                const double* q_wc_init_xyzw /* nullable */, const double* p_wc_init /* nullable */, const int32_t* init_valid /* nullable */,
                                double focal_length_init, double distortion_init, const icc_camcal_options* options /* nullable */,
                                double* intrinsics /* max(10, n_params(model)) */, double* q_wc_xyzw, double* p_wc, double* view_reproj_error_px, int32_t* view_used,
                                icc_camcal_summary* summary /* nullable */);
/* Shutter of icc_calibrate_camera.  line_delay_s = 0 (the default) is the global shutter and leaves the calibration exactly as above.
 * line_delay_s > 0 is a rolling shutter with the model of icc_set_pose_rolling_shutter: corner c of view i is seen tau = uv_c.y * line_delay_s
 * after the frame and predicted from P(tau) = exp(-tau [w_i]x) (R_cw (X - c_wc) - tau u_i), with the view's camera-frame velocities (w_i, u_i)
 * at row 0 held fixed in every bundle adjustment (the internal initialiser's included).  The residual is project(K, P(tau)) - uv with the same
 * Huber loss; the per-view errors and the 5 px / 2 px view filters use it, and the reported poses are those at the frame times.  With
 * optimize_board_points the board points are refined with the corners at their row times.  The line delay itself is not estimated here.
 *   w_u given (6 per view: w, u):    one calibration with these velocities (fixed mode); frame_t_s may be NULL.
 *   w_u NULL, frame_t_s given:       automatic mode.  Round 0 is the global-shutter calibration; if it returns success = 0, that result is
 *                                    returned.  Otherwise two rounds follow, each: the pose step (icc_estimate_board_poses' driver with the
 *                                    handle's icc_set_pose_error, max_reproj_error = 0, min_points = 0) on all n_views views under the previous
 *                                    round's intrinsics and a rolling shutter with these view times, then a calibration with the same inputs
 *                                    and options and the velocities that pose step used.  A view the pose step could not place, or that had
 *                                    no neighbour in time, gets w = u = 0 (the global-shutter model).  Every round reads the board points
 *                                    the handle held when icc_calibrate_camera was called; the outputs, the summary and (optimize_board_points)
 *                                    the refined board points are the last round's.
 * A negative or non-finite delay, a negative or non-finite time, a non-finite velocity, or a positive delay with n_views <= 0 or with both
 * arrays NULL is ICC_ERR_INVALID_ARGUMENT; so is a later icc_calibrate_camera with another n_views.  Host state only (a host-only handle
 * accepts it); the handle's camera and its pose-step shutter are not changed, by this call or by the calibration. */
icc_status icc_set_camcal_rolling_shutter(icc_handle* h, double line_delay_s, int32_t n_views, const double* frame_t_s /* nullable */,
                                          const double* w_u /* 6 per view, nullable */);
/* The velocities the last rolling-shutter icc_calibrate_camera on this handle used: w_u[6 * n_views] = (w, u) per view, and
 * n_without_neighbours (nullable) = the valid views without a neighbour in its last pose step (0 in fixed mode).  ICC_ERR_STATE before any
 * such call; ICC_ERR_INVALID_ARGUMENT when n_views differs from that call's. */
icc_status icc_get_camcal_velocities(const icc_handle* h, int32_t n_views, double* w_u, int32_t* n_without_neighbours);

/* ---- upstream: static IMU biases, the `--imu_bias_file` input of the hot CLI ------------------------------------------------------------
 * python/get_imu_biases.py:36-53: gyroscope bias = mean of the gyroscope stream; accelerometer bias = mean of the accelerometer stream
 * after removing gravity along the axis with the largest mean magnitude, gravity = gravity_const * sign(mean) stored as float32 there
 * (np.zeros(..., dtype=np.float32), :43-44 -- the rounding is reproduced).  The two column sums are one reduction kernel on the GPU.
 * Parity of this step is pinned by the reference's own Python (tests/golden/make_imu_bias_golden.py runs the unmodified script). */
icc_status icc_estimate_imu_biases(icc_handle* h, int n, const double* accel_xyz, const double* gyro_xyz, double gravity_const,
                                   double accl_bias[3], double gyro_bias[3]);

/* ---- upstream: static multi-pose IMU intrinsics, the `--imu_intrinsics` input of the hot CLI ---------------------------------------------
 * StaticImuCalibrator::CalibrateAccGyro (src/core/static_imu_calibrator.cc:54-337; imu_tk, Tedaldi et al. ICRA 2014) behind
 * applications/static_imu_calibration.cc.  The accelerometer bias is first the mean of the initial static interval with g_mag removed
 * from its (signed) largest component; the windowed variance norm of the accelerometer (win_size samples) is compared with
 * th_mult x the norm of the initial interval's variance for th_mult = 1..10; each multiplier keeps its static intervals of at least
 * interval_n_samples samples and, with at least min_num_intervals of them, fits the 9-parameter accelerometer triad
 * (g_mag - |T K (a - b)|, lower-left misalignment zero) with Ceres' default Levenberg-Marquardt options.  The multiplier with the
 * smallest final cost wins (strict <; the costs sum over different sample counts, as in the reference).  The gyroscope triad (9
 * parameters, 12 with optimize_gyro_bias) is then fitted on the RK4-integrated rotations between consecutive static poses, the
 * gyroscope bias being the mean of the initial interval (plus the fitted correction).  Timestamps must be non-decreasing and are
 * shared by both streams.
 * Outputs: acc_params [misYZ, misZY, misZX, sX, sY, sZ, bX, bY, bZ]; gyr_params [misYZ, misZY, misZX, misXZ, misXY, misYX, sX, sY, sZ]
 * (the order of icc_init_params' intrinsics); gyr_bias.  When no multiplier has enough intervals the reference's CalibrateAccGyro
 * returns false and its application still writes the default triads: the status is ICC_OK, summary->success = 0 and the outputs
 * are the identity triads with zero biases. */
typedef struct icc_static_imu_options {
  double g_mag;                      /* SetGravityMagnitude; 9.81 (the application passes --gravity_magnitude = 9.811107) */
  double init_interval_duration_s;   /* SetInitStaticIntervalDuration; 30 (the application passes --initial_static_interval_s = 10) */
  double gyro_dt;                    /* SetGyroDataPeriod; <= 0 integrates with the timestamp differences (default -1) */
  double init_acc[6];                /* SetInitAccCalibration: [misYZ, misZY, misZX, sX, sY, sZ]; default 0, 0, 0, 1, 1, 1 */
  double init_gyr[9];                /* SetInitGyroCalibration: gyr_params order; default 0 x 6, 1, 1, 1 */
  int32_t interval_n_samples;        /* SetIntarvalsNumSamples; 100 */
  int32_t min_num_intervals;         /* 12 */
  int32_t win_size;                  /* StaticIntervalsDetector window; 101 (at least 11, made odd) */
  int32_t acc_use_means;             /* EnableAccUseMeans; 0 */
  int32_t optimize_gyro_bias;        /* EnableGyroBiasOptimization; 0 */
  int32_t reserved;
} icc_static_imu_options;
typedef struct icc_static_imu_summary {
  int32_t success;                   /* CalibrateAccGyro's return value */
  int32_t chosen_multiplier;         /* 1..10, 0 when none qualified */
  int32_t n_intervals[10];           /* kept static intervals per multiplier */
  int32_t acc_iterations[10];        /* LM iterations per multiplier (0 when skipped) */
  int32_t acc_termination[10];       /* icc_summary.termination codes */
  int32_t gyro_iterations, gyro_termination;
  int32_t n_transitions;             /* consecutive static pose pairs in the gyroscope fit */
  int32_t gpu_launches;
  double norm_threshold;             /* norm of the initial interval's accelerometer variance */
  double acc_initial_cost[10], acc_final_cost[10];
  double acc_params[10][9];          /* fitted accelerometer parameters per multiplier */
  double gyro_initial_cost, gyro_final_cost;
  double seconds_total;              /* host wall clock of the call */
} icc_static_imu_summary;
void icc_default_static_imu_options(icc_static_imu_options* o);
icc_status icc_static_imu_calibration(icc_handle* h, int n, const double* t_s, const double* accel_xyz, const double* gyro_xyz,
                                      const icc_static_imu_options* options /* nullable */, double acc_params[9], double gyr_params[9],
                                      double gyr_bias[3], icc_static_imu_summary* summary /* nullable */);
/* Kept static intervals of the last icc_static_imu_calibration (inspection / tests): for each multiplier 1..10 its count, then that
 * many (start, end) sample index pairs (inclusive).  `buf` NULL returns the required length in *len; otherwise *len is its capacity. */
icc_status icc_get_static_imu_intervals(const icc_handle* h, int32_t* buf, int32_t* len);

/* ---- upstream: Allan variance noise characterisation of a static IMU log ----------------------------------------------------------------
 * AllanVarianceFitter::RunFit (src/core/allan_variance_fitter.cc; imu_utils) behind applications/fit_allan_variance.cc.  Channels are
 * 0-2 accelerometer x, y, z (m/s^2, used as given) and 3-5 gyroscope x, y, z (rad/s, scaled by 57.3 * 3600 to deg/h as pushRadPerSec
 * does).  With dt the mean timestamp difference, freq = 1/dt and theta = cumsum(x) / freq, the overlapping Allan variance
 *   sigma2(m) = sum_{k < n-2m} (theta[k+2m] - 2 theta[k+m] + theta[k])^2 / (2 (dt m)^2 (n - 2m)),   tau(m) = dt m,
 * is computed at the reference's cluster sizes m (n_clusters log-spaced values up to the largest power of two <= n/2, rounded up,
 * consecutive duplicates dropped).  Each channel then fits log10(Q^2/tau^2 + N^2/tau + B^2 + K^2 tau + R^2 tau^2) to log10(sigma2)
 * with Ceres' DOGLEG strategy and default options from the reference's least-squares initial values; the accelerometer fit drops
 * the points below tau = 1 s that raise the running maximum of sigma2 (FitAllanAcc::checkData).  params: [Q, N, B, K, R] per channel.
 * Deviation: the reference divides by zero for n < 3 or n_clusters < 2; here those return ICC_ERR_INVALID_ARGUMENT. */
typedef struct icc_allan_options {
  int32_t n_clusters;                /* log-spaced cluster sizes before deduplication; 10000 (fit_allan_variance.cc:41) */
  int32_t reserved;
} icc_allan_options;
typedef struct icc_allan_noise {     /* the quantities the reference prints per channel */
  double mean;                       /* gyroscope: mean rate in deg/s (getAvgValue() / 3600); accelerometer: mean in m/s^2 */
  double bias_instability;           /* min of the fitted deviation over the fitted taus (from 1000): rad/s (/ (57.3 * 3600)) or m/s^2 */
  double bias_instability_tau;       /* the tau of that minimum [s] */
  double bias_b;                     /* gyroscope: getB() / (57.3 * 3600) = |B| / 0.6642824703 / (57.3 * 3600) rad/s; 0 for the accelerometer */
  double white_noise_n;              /* gyroscope: sqrt(freq) getN() 60 / 57.3 = sqrt(freq) |N| / 57.3 rad/s; 0 for the accelerometer */
  double white_noise;                /* sqrt(freq) sqrt(model(tau = 1)): rad/s (/ (57.3 * 3600)) or m/s^2 */
} icc_allan_noise;
typedef struct icc_allan_summary {
  int32_t n_samples;
  int32_t n_factors;                 /* F: distinct cluster sizes */
  int32_t n_fit_points;              /* points in the fit (F, or fewer for the accelerometer) */
  int32_t iterations, successful_steps;
  int32_t termination;               /* icc_summary.termination codes */
  int32_t gpu_launches;              /* kernel launches of the whole call */
  int32_t reserved;
  double freq, period;               /* 1 / mean dt [Hz], mean dt [s] */
  double init_coeffs[5];             /* the signed least-squares solution initValue prints ("C ..."); the fit starts from |C| */
  double initial_cost, final_cost;
  double seconds_total;              /* host wall clock of the whole call (all channels) */
} icc_allan_summary;
void icc_default_allan_options(icc_allan_options* o);
icc_status icc_allan_variance(icc_handle* h, int n, const double* t_s, const double* accel_xyz, const double* gyro_xyz,
                              const icc_allan_options* options /* nullable */, double params[30] /* 6 x 5 */, icc_allan_noise noise[6],
                              icc_allan_summary summary[6]);
/* Curves of the last icc_allan_variance for one channel (0-5): factors, tau [s], sigma2 and the fitted deviation sqrt(model(tau)) at
 * every factor.  `factors` NULL returns F in *len; otherwise *len is the capacity of each array. */
icc_status icc_get_allan_curves(const icc_handle* h, int channel, int32_t* factors, double* tau, double* sigma2, double* fit_deviation, int32_t* len);

/* ---- upstream: radon checkerboard corners (extract_board_to_json --board_type radon) ---------------------------------------------------
 * BoardExtractor::ExtractBoard for BoardType::RADON (src/core/board_extractor.cc): cv::resize(frame, 1/f, INTER_LINEAR), then
 * cv::findChessboardCornersSB(CALIB_CB_LARGER | CALIB_CB_MARKER | CALIB_CB_EXHAUSTIVE) on the board of resource/checkerboard_radon.png
 * (corners_x x corners_y inner corners, 14 x 9 for the printed board, three circle markers next to the centre).  frames: n_frames 8-bit
 * gray images of width x height, row pitch pitch_bytes, frame k at frames + k height pitch_bytes, in host or device memory (detected
 * with cudaPointerGetAttributes; device frames are not copied through the host).  A frame is found iff exactly corners_x x
 * corners_y corners form one grid and the three markers sit in their squares; then uv_out holds its corners in the downsampled
 * image's pixels in id order id = i corners_x + j (row i, column j; the reference's continuous_board_indices_), in the corner order
 * findChessboardCornersSB returns.  Frames that are not found get found = 0 and their uv_out is left untouched.
 * ICC_ERR_INVALID_ARGUMENT, with nothing launched: corners_x or corners_y < 3, a factor < 1 or not finite, pitch < width, a NULL
 * frame or output pointer. */
typedef struct icc_board_summary {
  int32_t width, height;             /* the downsampled frame size */
  int32_t n_found;
  int32_t n_no_grid;                 /* too few candidates, or no grid grew from the seed */
  int32_t n_wrong_count;             /* the grid is not exactly corners_x x corners_y (a partial or a larger board) */
  int32_t n_no_markers;              /* the grid is complete but the three markers are not where the board has them */
  int64_t candidate_overflow;        /* candidates dropped because a frame's list (1024) was full, summed over the frames */
  int32_t gpu_launches;
  int32_t reserved;
  double seconds;                    /* host wall clock of the call */
} icc_board_summary;
icc_status icc_extract_radon_board(icc_handle* h, int n_frames, int width, int height, int64_t pitch_bytes, const uint8_t* frames, int corners_x,
                                   int corners_y, double downsample_factor, double* uv_out /* n_frames * corners_x * corners_y * 2 */,
                                   int32_t* found /* n_frames */, icc_board_summary* summary /* nullable */);
/* The same for colour frames: rows hold width interleaved B, G, R bytes (cv::imread's order), pitch_bytes >= 3 width.  The first stage is the
 * reference's order, cv::resize of the colour image (each channel as icc_extract_radon_board resizes gray) and then cv::cvtColor(BGR2GRAY)
 * with OpenCV's 15-bit rule (B 3735 + G 19235 + R 9798 + 16384) >> 15; at a factor of 1 only the conversion.  Every later step, the
 * argument checks, the chunking and the summary are those of icc_extract_radon_board.  A gray frame replicated to B = G = R gives the
 * same corners through either entry. */
icc_status icc_extract_radon_board_bgr(icc_handle* h, int n_frames, int width, int height, int64_t pitch_bytes, const uint8_t* frames_bgr, int corners_x,
                                       int corners_y, double downsample_factor, double* uv_out /* n_frames * corners_x * corners_y * 2 */,
                                       int32_t* found /* n_frames */, icc_board_summary* summary /* nullable */);
/* ---- upstream: Kalibr AprilGrid corners (extract_board_to_json --board_type apriltag) ------------------------------------------------
 * BoardExtractor::ExtractBoard for BoardType::APRILTAG (src/core/board_extractor.cc): cv::resize(frame, 1/f, INTER_LINEAR), then the
 * Kalibr/Basalt wrapper ApriltagDetector::detectTags (third_party/apriltag/apriltag.cpp) on tag36h11 with a 2-bit black border.  The board
 * has tags_x x tags_y tags; tag t = tags_x y + x has its corners i = 0..3 (bottom-left, bottom-right, top-right, top-left with the
 * board's y up) at point id (t << 2) + i.  frames: n_frames 8-bit gray images as for icc_extract_radon_board (host or device memory).
 * Per frame and point id (n_frames x 4 tags_x tags_y): uv_out (x, y) in the downsampled image's pixels and status_out 1 (kept),
 * 0 (not seen; uv NaN) or -1 (seen, but cornerSubPix moved it further than the wrapper's radius; uv is where it moved to).
 * found[k] = 1 iff frame k gives a view: it has >= 4 tags left after the wrapper's rules, in this order: a corner within 4 px of the
 * border, a Hamming distance > 1, an id >= 36 (the wrapper's limit whatever the board size), and no id appears twice.  A tag with an
 * id the board does not have (tags_x tags_y <= id < 36) counts for those rules but has no point ids.  Frames that are not found have
 * every status 0.  ICC_ERR_INVALID_ARGUMENT, with nothing launched: tags_x or tags_y outside 1..64, a factor < 1 or not finite,
 * pitch < width, a NULL frame or output pointer. */
typedef struct icc_aprilgrid_summary {
  int32_t width, height;             /* the downsampled frame size */
  int32_t n_found;                   /* frames with a view */
  int32_t n_few_tags;                /* frames with fewer than 4 tags after the tag rules */
  int32_t n_duplicate;               /* frames dropped because an id appeared twice */
  int32_t n_quads;                   /* dark components examined, summed over the frames */
  int32_t n_not_decoded;             /* quads whose 36 bits were not all inside the image */
  int32_t n_border;                  /* decoded tags dropped: a corner within 4 px of the border */
  int32_t n_not_good;                /* decoded tags dropped: Hamming distance > 1 (most quads that are not tags) */
  int32_t n_id_range;                /* decoded tags dropped: id >= 36 */
  int32_t n_corners_kept;            /* status 1 */
  int32_t n_corners_moved;           /* status -1 */
  int64_t quad_overflow;             /* components dropped because a frame's 1024 quad slots were full */
  int32_t gpu_launches;
  int32_t reserved;
  double seconds;                    /* host wall clock of the call */
} icc_aprilgrid_summary;
icc_status icc_extract_aprilgrid(icc_handle* h, int n_frames, int width, int height, int64_t pitch_bytes, const uint8_t* frames, int tags_x, int tags_y,
                                 double downsample_factor, double* uv_out /* n_frames * 4 tags_x tags_y * 2 */,
                                 int32_t* status_out /* n_frames * 4 tags_x tags_y */, int32_t* found /* n_frames */,
                                 icc_aprilgrid_summary* summary /* nullable */);
/* Page-locked host memory (cudaHostAlloc) for frames that a host program fills and hands to the extraction entries; *p = NULL for 0 bytes.
 * ICC_ERR_NO_DEVICE without a GPU, ICC_ERR_CUDA when the allocation fails.  Free with icc_host_free_pinned (NULL is accepted). */
icc_status icc_host_alloc_pinned(uint64_t bytes, void** p);
icc_status icc_host_free_pinned(void* p);

/* Device blocks of destroyed handles are cached process-wide for the next job; this returns them to the CUDA driver. */
void icc_trim_device_cache(void);

#ifdef __cplusplus
}
#endif
#endif /* ICC_B200_H_ */
