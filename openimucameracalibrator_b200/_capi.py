"""ctypes binding of the C-ABI declared in include/icc_b200.h.

`CApi(lib, prefix)` binds every entry point of a loaded shared library; the product binds `libicc_b200.so` with prefix
`icc_`.  (tests/ bind the CPU oracle, which deliberately exports the same shapes under `icco_`, through the same class —
the product package itself never loads or references the oracle.)
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .camera_models import MAX_INTRINSICS

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)
c_int64_p = C.POINTER(C.c_int64)

FLAG_POINTS, FLAG_T_I_C, FLAG_IMU_BIASES, FLAG_IMU_INTRINSICS = 1, 2, 4, 8
FLAG_GRAVITY_DIR, FLAG_CAM_LINE_DELAY, FLAG_SPLINE, FLAG_ACC_BIAS, FLAG_GYR_BIAS = 16, 32, 64, 128, 256
FLAG_CAM_INTRINSICS, FLAG_TIME_OFFSET = 512, 1024     # north-star extensions (the reference keeps both fixed)
POSE_ERROR_NORMALIZED, POSE_ERROR_TANGENT = 0, 1       # residual of the per-view pose step (icc_set_pose_error)
POSE_ERRORS = {"normalized": POSE_ERROR_NORMALIZED, "tangent": POSE_ERROR_TANGENT}
REPROJ_ERROR_PIXEL, REPROJ_ERROR_TANGENT = 0, 1         # vision residual of the spline solve (icc_set_reprojection_error)
REPROJ_ERRORS = {"pixel": REPROJ_ERROR_PIXEL, "tangent": REPROJ_ERROR_TANGENT}

STATUS_NAMES = {0: "ICC_OK", 1: "ICC_ERR_INVALID_ARGUMENT", 2: "ICC_ERR_NO_DEVICE", 3: "ICC_ERR_CUDA", 4: "ICC_ERR_STATE",
                5: "ICC_ERR_UNSUPPORTED", 6: "ICC_ERR_NUMERIC"}
TERMINATION = {0: "max_iterations", 1: "function_tolerance", 2: "parameter_tolerance", 3: "gradient_tolerance", 4: "failure"}


class InitParams(C.Structure):
    _fields_ = [("T_i_c_init", C.c_double * 7), ("dt_so3_s", C.c_double), ("dt_r3_s", C.c_double), ("std_so3", C.c_double),
                ("std_r3", C.c_double), ("time_offset_imu_to_cam_s", C.c_double), ("init_line_delay_s", C.c_double),
                ("acc_intrinsics", C.c_double * 6), ("gyr_intrinsics", C.c_double * 9), ("acc_bias", C.c_double * 3),
                ("gyr_bias", C.c_double * 3), ("dispatch_fov", C.c_int32), ("reserved", C.c_int32)]


class SolverOptions(C.Structure):
    _fields_ = [("function_tolerance", C.c_double), ("parameter_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double), ("min_lm_diagonal", C.c_double),
                ("max_lm_diagonal", C.c_double), ("jacobi_scaling", C.c_int32), ("max_consecutive_invalid_steps", C.c_int32)]


class Summary(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("successful_steps", C.c_int32), ("termination", C.c_int32), ("num_residuals", C.c_int32),
                ("num_tangent", C.c_int32), ("jacobian_evaluations", C.c_int32), ("cost_evaluations", C.c_int32),
                ("gpu_launches", C.c_int32), ("initial_cost", C.c_double), ("final_cost", C.c_double),
                ("mean_reproj_error", C.c_double), ("seconds_total", C.c_double), ("seconds_jacobian", C.c_double),
                ("seconds_linear_solve", C.c_double)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["termination_name"] = TERMINATION.get(self.termination, "?")
        return d


class OutlierSummary(C.Structure):
    """icc_outlier_summary (include/icc_b200.h): what one icc_reject_outlier_corners call did, summed over the shards."""
    _fields_ = [("n_corners", C.c_int64), ("n_rejected", C.c_int64), ("n_failed", C.c_int64), ("n_frames_emptied", C.c_int32),
                ("reserved", C.c_int32), ("rms_px", C.c_double), ("threshold_px", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class CamCalOptions(C.Structure):
    """icc_camcal_options (include/icc_b200.h): zero / negative fields select the reference's defaults."""
    _fields_ = [("grid_size", C.c_double), ("function_tolerance", C.c_double), ("parameter_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("huber_width", C.c_double), ("max_view_error_stage1_px", C.c_double), ("max_view_error_final_px", C.c_double),
                ("min_num_views", C.c_int32), ("max_num_iterations", C.c_int32), ("optimize_board_points", C.c_int32), ("reserved", C.c_int32)]


class CamCalSummary(C.Structure):
    _fields_ = [("success", C.c_int32), ("n_views_initialized", C.c_int32), ("n_views_selected", C.c_int32), ("n_views_used", C.c_int32),
                ("iterations", C.c_int32 * 3), ("termination", C.c_int32 * 3), ("gpu_launches", C.c_int32), ("init_iterations", C.c_int32), ("n_points_optimized", C.c_int32), ("reserved", C.c_int32),
                ("focal_length_init", C.c_double), ("initial_cost", C.c_double), ("final_cost", C.c_double * 3), ("final_reproj_error", C.c_double),
                ("seconds_total", C.c_double)]

    def as_dict(self):
        d = {}
        for k, _ in self._fields_:
            v = getattr(self, k)
            d[k] = list(v) if hasattr(v, "__len__") else v
        return d


class StaticImuOptions(C.Structure):
    """icc_static_imu_options (include/icc_b200.h); icc_default_static_imu_options fills in the reference's defaults."""
    _fields_ = [("g_mag", C.c_double), ("init_interval_duration_s", C.c_double), ("gyro_dt", C.c_double), ("init_acc", C.c_double * 6),
                ("init_gyr", C.c_double * 9), ("interval_n_samples", C.c_int32), ("min_num_intervals", C.c_int32), ("win_size", C.c_int32),
                ("acc_use_means", C.c_int32), ("optimize_gyro_bias", C.c_int32), ("reserved", C.c_int32)]


class StaticImuSummary(C.Structure):
    _fields_ = [("success", C.c_int32), ("chosen_multiplier", C.c_int32), ("n_intervals", C.c_int32 * 10), ("acc_iterations", C.c_int32 * 10),
                ("acc_termination", C.c_int32 * 10), ("gyro_iterations", C.c_int32), ("gyro_termination", C.c_int32), ("n_transitions", C.c_int32),
                ("gpu_launches", C.c_int32), ("norm_threshold", C.c_double), ("acc_initial_cost", C.c_double * 10), ("acc_final_cost", C.c_double * 10),
                ("acc_params", (C.c_double * 9) * 10), ("gyro_initial_cost", C.c_double), ("gyro_final_cost", C.c_double), ("seconds_total", C.c_double)]

    def as_dict(self):
        d = {}
        for k, _ in self._fields_:
            v = getattr(self, k)
            d[k] = np.array([list(r) for r in v]) if k == "acc_params" else (list(v) if hasattr(v, "__len__") else v)
        return d


class AllanOptions(C.Structure):
    """icc_allan_options (include/icc_b200.h); icc_default_allan_options fills in the reference's defaults."""
    _fields_ = [("n_clusters", C.c_int32), ("reserved", C.c_int32)]


class AllanNoise(C.Structure):
    _fields_ = [("mean", C.c_double), ("bias_instability", C.c_double), ("bias_instability_tau", C.c_double), ("bias_b", C.c_double),
                ("white_noise_n", C.c_double), ("white_noise", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class AllanSummary(C.Structure):
    _fields_ = [("n_samples", C.c_int32), ("n_factors", C.c_int32), ("n_fit_points", C.c_int32), ("iterations", C.c_int32),
                ("successful_steps", C.c_int32), ("termination", C.c_int32), ("gpu_launches", C.c_int32), ("reserved", C.c_int32),
                ("freq", C.c_double), ("period", C.c_double), ("init_coeffs", C.c_double * 5), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("seconds_total", C.c_double)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["init_coeffs"] = list(self.init_coeffs)
        return d


ALLAN_CHANNELS = ("acc_x", "acc_y", "acc_z", "gyr_x", "gyr_y", "gyr_z")
ALLAN_PARAMS = ("Q", "N", "B", "K", "R")

ALLREDUCE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p)


class IccError(RuntimeError):
    pass


def _dp(a):
    return None if a is None else a.ctypes.data_as(c_double_p)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class BoardSummary(C.Structure):
    """icc_board_summary (include/icc_b200.h): what one icc_extract_radon_board call did."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("n_found", C.c_int32), ("n_no_grid", C.c_int32), ("n_wrong_count", C.c_int32),
                ("n_no_markers", C.c_int32), ("candidate_overflow", C.c_int64), ("gpu_launches", C.c_int32), ("reserved", C.c_int32),
                ("seconds", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class AprilGridSummary(C.Structure):
    """icc_aprilgrid_summary (include/icc_b200.h): what one icc_extract_aprilgrid call did."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("n_found", C.c_int32), ("n_few_tags", C.c_int32), ("n_duplicate", C.c_int32),
                ("n_quads", C.c_int32), ("n_not_decoded", C.c_int32), ("n_border", C.c_int32), ("n_not_good", C.c_int32), ("n_id_range", C.c_int32),
                ("n_corners_kept", C.c_int32), ("n_corners_moved", C.c_int32), ("quad_overflow", C.c_int64), ("gpu_launches", C.c_int32),
                ("reserved", C.c_int32), ("seconds", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


def _frames_pointer(frames):
    """(pointer, n, height, width, pitch in bytes) of 8-bit frames: an (N, H, W) or (H, W) uint8 NumPy array, or a torch CUDA tensor,
    whose rows are contiguous and whose frames are `height` rows of one pitch apart."""
    if hasattr(frames, "data_ptr"):   # torch tensor: passed by pointer, never copied through the host
        t = frames if frames.dim() == 3 else frames.unsqueeze(0)
        assert str(t.dtype) == "torch.uint8", t.dtype
        n, h, w = t.shape
        s0, s1, s2 = t.stride()
        ptr = t.data_ptr()
    else:
        a = np.asarray(frames)
        if a.ndim == 2:
            a = a[None]
        assert a.dtype == np.uint8, a.dtype
        n, h, w = a.shape
        s0, s1, s2 = a.strides
        ptr = a.ctypes.data
    if s2 != 1 or (n > 1 and s0 != h * s1) or s1 < w:
        raise ValueError("frames need contiguous rows, one row pitch >= width, and frames `height` rows apart")
    return ptr, n, h, w, s1


def _bgr_frames_pointer(frames):
    """(pointer, n, height, width, pitch in bytes) of 8-bit B, G, R frames: an (N, H, W, 3) or (H, W, 3) uint8 NumPy array, or a torch CUDA
    tensor, whose pixels are interleaved and contiguous along each row and whose frames are `height` rows of one pitch apart."""
    if hasattr(frames, "data_ptr"):
        t = frames if frames.dim() == 4 else frames.unsqueeze(0)
        assert str(t.dtype) == "torch.uint8", t.dtype
        n, h, w, c = t.shape
        s0, s1, s2, s3 = t.stride()
        ptr = t.data_ptr()
    else:
        a = np.asarray(frames)
        if a.ndim == 3:
            a = a[None]
        assert a.dtype == np.uint8, a.dtype
        n, h, w, c = a.shape
        s0, s1, s2, s3 = a.strides
        ptr = a.ctypes.data
    if c != 3 or s3 != 1 or s2 != 3 or (n > 1 and s0 != h * s1) or s1 < 3 * w:
        raise ValueError("colour frames need 3 interleaved channels, contiguous rows, one row pitch >= 3 width, and frames `height` rows apart")
    return ptr, n, h, w, s1


class CApi:
    """Thin object wrapper around one solver handle of a loaded library."""

    def __init__(self, lib: C.CDLL, prefix: str, create_arg: int = 0):
        self.lib, self.prefix = lib, prefix
        self._keepalive = []
        h = C.c_void_p()
        f = self._fn("create"); f.restype = C.c_int; f.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        st = f(C.byref(h), create_arg)
        self.h = h
        if st != 0:
            msg = self.last_error() if h.value else ""
            self.h = None
            raise IccError(f"{prefix}create failed: {STATUS_NAMES.get(st, st)} {msg}")

    def _fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def last_error(self) -> str:
        f = self._fn("last_error"); f.restype = C.c_char_p; f.argtypes = [C.c_void_p]
        return (f(self.h) or b"").decode()

    def _call(self, name, argtypes, *args):
        f = self._fn(name); f.restype = C.c_int; f.argtypes = [C.c_void_p] + list(argtypes)
        st = f(self.h, *args)
        if st != 0:
            raise IccError(f"{self.prefix}{name}: {STATUS_NAMES.get(st, st)}: {self.last_error()}")

    def close(self):
        if getattr(self, "h", None):
            f = self._fn("destroy"); f.restype = None; f.argtypes = [C.c_void_p]
            f(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- problem data --------------------------------------------------------------------------------------
    def set_solver_options(self, **kw):
        o = default_solver_options()
        for k, v in kw.items():
            setattr(o, k, v)
        self._call("set_solver_options", [C.POINTER(SolverOptions)], C.byref(o))

    def set_camera(self, model, intrinsics, width, height):
        k = _f64(intrinsics)
        self._call("set_camera", [C.c_int, c_double_p, C.c_int, C.c_int, C.c_int], int(model), _dp(k), k.size, int(width), int(height))

    def set_board_points(self, xyzw):
        p = _f64(xyzw).reshape(-1, 4)
        self._n_board = p.shape[0]
        self._call("set_board_points", [C.c_int, c_double_p], p.shape[0], _dp(p))

    def set_frames(self, t_s, corner_offsets, point_ids, uv, q_wc, p_wc):
        t = _f64(t_s); off = np.ascontiguousarray(corner_offsets, dtype=np.int32); ids = np.ascontiguousarray(point_ids, dtype=np.int32)
        uv = _f64(uv); q = _f64(q_wc); p = _f64(p_wc)
        assert off.size == t.size + 1 and ids.size == off[-1] and uv.size == 2 * ids.size and q.size == 4 * t.size and p.size == 3 * t.size
        self._n_corners_in = int(ids.size)
        self._call("set_frames", [C.c_int, c_double_p, c_int32_p, c_int32_p, c_double_p, c_double_p, c_double_p], t.size, _dp(t),
                   off.ctypes.data_as(c_int32_p), ids.ctypes.data_as(c_int32_p), _dp(uv), _dp(q), _dp(p))

    def set_imu(self, t_s, accel, gyro):
        t = _f64(t_s); a = _f64(accel); g = _f64(gyro)
        assert a.size == 3 * t.size and g.size == 3 * t.size
        self._call("set_imu", [C.c_int, c_double_p, c_double_p, c_double_p], t.size, _dp(t), _dp(a), _dp(g))

    # ---- upstream row f1: per-view board poses (PoseEstimator::EstimatePosesFromJson, src/core/pose_estimator.cc:92-191) ----
    def estimate_board_poses(self, corner_offsets, point_ids, uv, max_reproj_error=0.0, min_points=0):
        """-> (q_wc[n,4] x,y,z,w, p_wc[n,3], mean normalised reprojection error[n], valid[n]); camera + board points must be set."""
        off = np.ascontiguousarray(corner_offsets, dtype=np.int32); ids = np.ascontiguousarray(point_ids, dtype=np.int32); uv = _f64(uv)
        n = off.size - 1
        assert ids.size == off[-1] and uv.size == 2 * ids.size
        q = np.zeros((n, 4)); p = np.zeros((n, 3)); e = np.zeros(n); v = np.zeros(n, dtype=np.int32)
        self._call("estimate_board_poses", [C.c_int, c_int32_p, c_int32_p, c_double_p, C.c_double, C.c_int, c_double_p, c_double_p, c_double_p, c_int32_p],
                   n, off.ctypes.data_as(c_int32_p), ids.ctypes.data_as(c_int32_p), _dp(uv), float(max_reproj_error), int(min_points),
                   _dp(q), _dp(p), _dp(e), v.ctypes.data_as(c_int32_p))
        return q, p, e, v

    def filter_bad_poses(self, p_wc, valid):
        """PoseEstimator::FilterBadPoses (src/core/pose_estimator.cc:238-261): -> valid with the outlying camera heights cleared."""
        p = _f64(p_wc).reshape(-1, 3); v = np.array(valid, dtype=np.int32)
        self._call("filter_bad_poses", [C.c_int, c_double_p, c_int32_p], p.shape[0], _dp(p), v.ctypes.data_as(c_int32_p))
        return v

    def optimize_board_points(self, corner_offsets, point_ids, uv, q_wc, p_wc, valid, max_reproj_error=0.0, min_points=0, min_observations=0):
        """PoseEstimator::OptimizeBoardPoints + OptimizeAllPoses (pose_estimator.cc:193-236)
        -> (q_wc, p_wc, mean error, valid, board_xyzw, number of optimised points); the handle's board points are replaced."""
        off = np.ascontiguousarray(corner_offsets, dtype=np.int32); ids = np.ascontiguousarray(point_ids, dtype=np.int32); uv = _f64(uv)
        n = off.size - 1
        q = np.array(q_wc, dtype=np.float64).reshape(n, 4).copy(); p = np.array(p_wc, dtype=np.float64).reshape(n, 3).copy()
        v = np.array(valid, dtype=np.int32).copy(); e = np.zeros(n); nopt = C.c_int32()
        board = np.zeros((self.num_board_points(), 4))
        self._call("optimize_board_points", [C.c_int, c_int32_p, c_int32_p, c_double_p, C.c_double, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p, c_int32_p, c_double_p, C.POINTER(C.c_int32)],
                   n, off.ctypes.data_as(c_int32_p), ids.ctypes.data_as(c_int32_p), _dp(uv), float(max_reproj_error), int(min_points), int(min_observations),
                   _dp(q), _dp(p), _dp(e), v.ctypes.data_as(c_int32_p), _dp(board), C.byref(nopt))
        return q, p, e, v, board, nopt.value

    def num_board_points(self):
        return getattr(self, "_n_board", 0)

    def get_board_points(self):
        b = np.zeros((self.num_board_points(), 4)); self._call("get_board_points", [c_double_p, C.c_int], _dp(b), b.shape[0]); return b

    def pixels_to_normalized(self, uv):
        """theia::Camera::PixelToNormalizedCoordinates / z for an (n, 2) pixel array -> (xy[n,2], ok[n])."""
        uv = _f64(uv).reshape(-1, 2); n = uv.shape[0]
        xy = np.zeros((n, 2)); ok = np.zeros(n, dtype=np.int32)
        self._call("pixels_to_normalized", [C.c_int, c_double_p, c_double_p, c_int32_p], n, _dp(uv), _dp(xy), ok.ctypes.data_as(c_int32_p))
        return xy, ok

    def pixels_to_bearings(self, uv):
        """Unit bearing vectors of an (n, 2) pixel array -> (xyz[n,3], ok[n]); rays past 90 degrees where the camera model has them."""
        uv = _f64(uv).reshape(-1, 2); n = uv.shape[0]
        xyz = np.zeros((n, 3)); ok = np.zeros(n, dtype=np.int32)
        self._call("pixels_to_bearings", [C.c_int, c_double_p, c_double_p, c_int32_p], n, _dp(uv), _dp(xyz), ok.ctypes.data_as(c_int32_p))
        return xyz, ok

    def set_pose_error(self, mode):
        """Residual of estimate_board_poses / optimize_board_points: POSE_ERROR_NORMALIZED (default), POSE_ERROR_TANGENT, or their names."""
        self._call("set_pose_error", [C.c_int], POSE_ERRORS[mode] if isinstance(mode, str) else int(mode))

    def set_reprojection_error(self, mode):
        """Vision residual of the spline solve, before batch_init_spline: REPROJ_ERROR_PIXEL (default), REPROJ_ERROR_TANGENT (the local
        tangent reprojection error on the corners' bearings), or their names "pixel" / "tangent"."""
        self._call("set_reprojection_error", [C.c_int], REPROJ_ERRORS[mode] if isinstance(mode, str) else int(mode))

    def set_pose_rolling_shutter(self, line_delay_s, frame_t_s=None):
        """Shutter of estimate_board_poses / optimize_board_points: line_delay_s = 0 is the global shutter (the default); > 0 a rolling
        shutter with the views' frame times frame_t_s (one per view of the next pose call)."""
        t = None if frame_t_s is None else _f64(frame_t_s).ravel()
        self._call("set_pose_rolling_shutter", [C.c_double, C.c_int32, c_double_p], float(line_delay_s), 0 if t is None else t.size, _dp(t))

    def pose_velocities(self, n_frames):
        """Velocities of the last rolling-shutter pose call -> (w[n,3] rad/s, u[n,3] m/s, both camera frame at the frame time,
        number of valid views without a neighbour)."""
        vel = np.zeros((int(n_frames), 6)); ns = C.c_int32()
        self._call("get_pose_velocities", [C.c_int32, c_double_p, C.POINTER(C.c_int32)], int(n_frames), _dp(vel), C.byref(ns))
        return vel[:, :3], vel[:, 3:], ns.value

    def set_camcal_rolling_shutter(self, line_delay_s, frame_t_s=None, w_u=None):
        """Shutter of calibrate_camera: line_delay_s = 0 is the global shutter (the default); > 0 a rolling shutter, either with the views'
        fixed camera-frame velocities w_u[n,6] = (w, u), or (w_u None) in automatic mode with the views' frame times frame_t_s."""
        t = None if frame_t_s is None else _f64(frame_t_s).ravel()
        v = None if w_u is None else _f64(w_u).reshape(-1, 6)
        n = v.shape[0] if v is not None else (t.size if t is not None else 0)
        if t is not None and v is not None and t.size != n:
            raise ValueError("frame_t_s and w_u must describe the same number of views")
        self._call("set_camcal_rolling_shutter", [C.c_double, C.c_int32, c_double_p, c_double_p], float(line_delay_s), n, _dp(t), _dp(v))

    def camcal_velocities(self, n_views):
        """Velocities of the last rolling-shutter calibrate_camera -> (w[n,3] rad/s, u[n,3] m/s, both camera frame at the frame time,
        number of valid views without a neighbour in its last pose step)."""
        vel = np.zeros((int(n_views), 6)); ns = C.c_int32()
        self._call("get_camcal_velocities", [C.c_int32, c_double_p, C.POINTER(C.c_int32)], int(n_views), _dp(vel), C.byref(ns))
        return vel[:, :3], vel[:, 3:], ns.value

    # ---- upstream row f4: CameraCalibrator::CalibrateCameraFromJson / RunCalibration (src/core/camera_calibrator.cc:131-389) ----
    def calibrate_camera(self, model, image_width, image_height, corner_offsets, point_ids, uv, q_wc_init=None, p_wc_init=None, init_valid=None,
                         focal_length_init=0.0, distortion_init=0.0, **options):
        """-> dict(intrinsics[n], q_wc[nv,4], p_wc[nv,3], view_error_px[nv], used[nv], summary); board points must be set.
        options: fields of icc_camcal_options (grid_size defaults to the reference's 0.04 m)."""
        off = np.ascontiguousarray(corner_offsets, dtype=np.int32); ids = np.ascontiguousarray(point_ids, dtype=np.int32); uv = _f64(uv)
        nv = off.size - 1
        assert ids.size == off[-1] and uv.size == 2 * ids.size
        o = CamCalOptions(); o.grid_size = -1.0
        for k, v in options.items():
            setattr(o, k, v)
        qi = None if q_wc_init is None else _f64(q_wc_init); pi = None if p_wc_init is None else _f64(p_wc_init)
        vi = None if init_valid is None else np.ascontiguousarray(init_valid, dtype=np.int32)
        intr = np.zeros(MAX_INTRINSICS); q = np.zeros((nv, 4)); p = np.zeros((nv, 3)); e = np.zeros(nv); used = np.zeros(nv, dtype=np.int32); s = CamCalSummary()
        self._call("calibrate_camera", [C.c_int, C.c_int, C.c_int, C.c_int, c_int32_p, c_int32_p, c_double_p, c_double_p, c_double_p, c_int32_p, C.c_double, C.c_double,
                                        C.POINTER(CamCalOptions), c_double_p, c_double_p, c_double_p, c_double_p, c_int32_p, C.POINTER(CamCalSummary)],
                   int(model), int(image_width), int(image_height), nv, off.ctypes.data_as(c_int32_p), ids.ctypes.data_as(c_int32_p), _dp(uv),
                   None if qi is None else _dp(qi), None if pi is None else _dp(pi), None if vi is None else vi.ctypes.data_as(c_int32_p),
                   float(focal_length_init), float(distortion_init), C.byref(o), _dp(intr), _dp(q), _dp(p), _dp(e), used.ctypes.data_as(c_int32_p), C.byref(s))
        from .camera_models import NUM_PARAMS
        return dict(intrinsics=intr[:NUM_PARAMS[int(model)]], q_wc=q, p_wc=p, view_error_px=e, used=used, summary=s.as_dict())

    # ---- upstream row f3: ImuToCameraRotationEstimator (src/core/imu_to_camera_rotation_estimator.cc:116-274) -----------------
    def estimate_imu_to_camera_rotation(self, view_t_s, q_cw_xyzw, imu_t_s, gyro, gyro_bias=None):
        """-> dict(q_gyro_to_cam (x,y,z,w), time_offset_s, gyro_bias[3], error, iterations); gyro_bias=None estimates the bias."""
        vt = _f64(view_t_s); q = _f64(q_cw_xyzw); it = _f64(imu_t_s); g = _f64(gyro)
        assert q.size == 4 * vt.size and g.size == 3 * it.size
        qo = np.zeros(4); td = C.c_double(); bo = np.zeros(3); err = C.c_double(); iters = C.c_int32()
        b = None if gyro_bias is None else _f64(gyro_bias)
        self._call("estimate_imu_to_camera_rotation", [C.c_int, c_double_p, c_double_p, C.c_int, c_double_p, c_double_p, c_double_p, c_double_p,
                                                       C.POINTER(C.c_double), c_double_p, C.POINTER(C.c_double), C.POINTER(C.c_int32)],
                   vt.size, _dp(vt), _dp(q), it.size, _dp(it), _dp(g), None if b is None else _dp(b), _dp(qo), C.byref(td), _dp(bo), C.byref(err), C.byref(iters))
        return dict(q_gyro_to_cam=qo, time_offset_s=td.value, gyro_bias=bo, error=err.value, iterations=iters.value)

    # ---- upstream: static IMU biases (python/get_imu_biases.py:36-53) -----------------------------------------------------------------
    def estimate_imu_biases(self, accel, gyro, gravity_const=9.81):
        """-> (accl_bias[3], gyro_bias[3]) as written to the hot CLI's --imu_bias_file."""
        a = _f64(accel).reshape(-1, 3); g = _f64(gyro).reshape(-1, 3)
        assert a.shape == g.shape
        ba, bg = np.zeros(3), np.zeros(3)
        self._call("estimate_imu_biases", [C.c_int, c_double_p, c_double_p, C.c_double, c_double_p, c_double_p], a.shape[0], _dp(a), _dp(g), float(gravity_const), _dp(ba), _dp(bg))
        return ba, bg

    # ---- upstream: static multi-pose IMU intrinsics (src/core/static_imu_calibrator.cc:54-337) -------------------------------------
    def static_imu_options(self, **kw) -> StaticImuOptions:
        """The reference's defaults with the given fields replaced (init_acc / init_gyr as sequences)."""
        o = StaticImuOptions()
        f = self._fn("default_static_imu_options"); f.restype = None; f.argtypes = [C.POINTER(StaticImuOptions)]
        f(C.byref(o))
        for k, v in kw.items():
            if k in ("init_acc", "init_gyr"):
                getattr(o, k)[:] = [float(x) for x in v]
            else:
                setattr(o, k, type(getattr(o, k))(v))
        return o

    def static_imu_calibration(self, t_s, accel, gyro, **options):
        """-> dict(acc_params[9], gyr_params[9], gyr_bias[3], summary); options are icc_static_imu_options fields."""
        t = _f64(t_s); a = _f64(accel).reshape(-1, 3); g = _f64(gyro).reshape(-1, 3)
        assert a.shape == g.shape and a.shape[0] == t.size
        o = self.static_imu_options(**options)
        ap, gp, gb, s = np.zeros(9), np.zeros(9), np.zeros(3), StaticImuSummary()
        self._call("static_imu_calibration", [C.c_int, c_double_p, c_double_p, c_double_p, C.POINTER(StaticImuOptions), c_double_p, c_double_p, c_double_p,
                                              C.POINTER(StaticImuSummary)], t.size, _dp(t), _dp(a), _dp(g), C.byref(o), _dp(ap), _dp(gp), _dp(gb), C.byref(s))
        return dict(acc_params=ap, gyr_params=gp, gyr_bias=gb, summary=s.as_dict())

    def static_imu_intervals(self):
        """Kept static intervals of the last static_imu_calibration: list of ten (k, 2) int arrays (inclusive start, end)."""
        n = C.c_int32()
        self._call("get_static_imu_intervals", [c_int32_p, C.POINTER(C.c_int32)], None, C.byref(n))
        buf = np.zeros(max(n.value, 1), dtype=np.int32)
        self._call("get_static_imu_intervals", [c_int32_p, C.POINTER(C.c_int32)], buf.ctypes.data_as(c_int32_p), C.byref(n))
        out, k = [], 0
        for _ in range(10):
            c = int(buf[k]); out.append(buf[k + 1:k + 1 + 2 * c].reshape(c, 2).astype(np.int64)); k += 1 + 2 * c
        return out

    # ---- upstream: Allan variance noise characterisation (src/core/allan_variance_fitter.cc) ------------------------------------
    def allan_variance(self, t_s, accel, gyro, n_clusters=None):
        """-> dict(params (6, 5) [Q, N, B, K, R], noise [6 dicts], summary [6 dicts]); channels ALLAN_CHANNELS."""
        t = _f64(t_s); a = _f64(accel).reshape(-1, 3); g = _f64(gyro).reshape(-1, 3)
        assert a.shape == g.shape and a.shape[0] == t.size
        o = AllanOptions()
        f = self._fn("default_allan_options"); f.restype = None; f.argtypes = [C.POINTER(AllanOptions)]
        f(C.byref(o))
        if n_clusters is not None:
            o.n_clusters = int(n_clusters)
        p, z, s = np.zeros(30), (AllanNoise * 6)(), (AllanSummary * 6)()
        self._call("allan_variance", [C.c_int, c_double_p, c_double_p, c_double_p, C.POINTER(AllanOptions), c_double_p, C.POINTER(AllanNoise),
                                      C.POINTER(AllanSummary)], t.size, _dp(t), _dp(a), _dp(g), C.byref(o), _dp(p), z, s)
        return dict(params=p.reshape(6, 5), noise=[x.as_dict() for x in z], summary=[x.as_dict() for x in s])

    def allan_curves(self, channel):
        """Curves of the last allan_variance for channel 0-5: dict(factors, tau, sigma2, fit_deviation)."""
        args = [C.c_int, c_int32_p, c_double_p, c_double_p, c_double_p, C.POINTER(C.c_int32)]
        n = C.c_int32()
        self._call("get_allan_curves", args, int(channel), None, None, None, None, C.byref(n))
        f = np.zeros(max(n.value, 1), dtype=np.int32); t, s2, d = (np.zeros(max(n.value, 1)) for _ in range(3))
        self._call("get_allan_curves", args, int(channel), f.ctypes.data_as(c_int32_p), _dp(t), _dp(s2), _dp(d), C.byref(n))
        k = n.value
        return dict(factors=f[:k].astype(np.int64), tau=t[:k], sigma2=s2[:k], fit_deviation=d[:k])

    # ---- upstream: radon checkerboard corners (src/core/board_extractor.cc, BoardType::RADON) ----------------------------------
    def extract_radon_board(self, frames, corners_x, corners_y, downsample_factor=1.0):
        """-> (uv (N, corners_y * corners_x, 2) in id order, NaN for frames not found, found (N,) bool, summary dict).  frames: (N, H, W)
        or (H, W) uint8 NumPy array, or a torch CUDA uint8 tensor (read on the device by pointer)."""
        ptr, n, h, w, pitch = _frames_pointer(frames)
        uv = np.full((n, corners_x * corners_y, 2), np.nan)
        found = np.zeros(n, dtype=np.int32)
        s = BoardSummary()
        self._call("extract_radon_board", [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_double, c_double_p, c_int32_p,
                                           C.POINTER(BoardSummary)], n, w, h, pitch, C.c_void_p(ptr), int(corners_x), int(corners_y),
                   float(downsample_factor), _dp(uv), found.ctypes.data_as(c_int32_p), C.byref(s))
        return uv, found.astype(bool), s.as_dict()

    def extract_radon_board_bgr(self, frames, corners_x, corners_y, downsample_factor=1.0):
        """extract_radon_board for colour frames, resized and then converted to gray as the reference does (icc_extract_radon_board_bgr).
        frames: (N, H, W, 3) or (H, W, 3) uint8 in B, G, R order (cv2.imread's), a NumPy array or a torch CUDA tensor."""
        ptr, n, h, w, pitch = _bgr_frames_pointer(frames)
        uv = np.full((n, corners_x * corners_y, 2), np.nan)
        found = np.zeros(n, dtype=np.int32)
        s = BoardSummary()
        self._call("extract_radon_board_bgr", [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_double, c_double_p, c_int32_p,
                                               C.POINTER(BoardSummary)], n, w, h, pitch, C.c_void_p(ptr), int(corners_x), int(corners_y),
                   float(downsample_factor), _dp(uv), found.ctypes.data_as(c_int32_p), C.byref(s))
        return uv, found.astype(bool), s.as_dict()

    # ---- upstream: Kalibr AprilGrid corners (src/core/board_extractor.cc, BoardType::APRILTAG) -----------------------------------
    def extract_aprilgrid(self, frames, tags_x=6, tags_y=6, downsample_factor=1.0):
        """-> (uv (N, 4 tags_x tags_y, 2) per point id (t << 2) + i, NaN where not seen, status (N, 4 tags_x tags_y) int32: 1 kept,
        0 not seen, -1 moved too far by the refinement, found (N,) bool, summary dict).  frames as for extract_radon_board."""
        ptr, n, h, w, pitch = _frames_pointer(frames)
        n_pts = 4 * int(tags_x) * int(tags_y)
        uv = np.full((n, n_pts, 2), np.nan)
        status = np.zeros((n, n_pts), dtype=np.int32)
        found = np.zeros(n, dtype=np.int32)
        s = AprilGridSummary()
        self._call("extract_aprilgrid", [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_double, c_double_p, c_int32_p,
                                         c_int32_p, C.POINTER(AprilGridSummary)], n, w, h, pitch, C.c_void_p(ptr), int(tags_x), int(tags_y),
                   float(downsample_factor), _dp(uv), status.ctypes.data_as(c_int32_p), found.ctypes.data_as(c_int32_p), C.byref(s))
        return uv, status, found.astype(bool), s.as_dict()

    # ---- upstream row f2: spline error weighting (python/sew.py:knot_spacing_and_variance) ------------------------------------
    def spline_error_weighting(self, times_s, signal_xyz, quality, min_dt=0.0, max_dt=0.0, want_spectrum=False):
        """-> (knot_spacing, variance[, reference spectrum Xhat]); signal_xyz is (n, 3)."""
        t = _f64(times_s); x = _f64(signal_xyz).reshape(-1, 3)
        assert x.shape[0] == t.size
        dt = C.c_double(); var = C.c_double(); spec = np.zeros(t.size) if want_spectrum else None
        self._call("spline_error_weighting", [C.c_int, c_double_p, c_double_p, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double), c_double_p],
                   t.size, _dp(t), _dp(x), float(quality), float(min_dt), float(max_dt), C.byref(dt), C.byref(var), None if spec is None else _dp(spec))
        return (dt.value, var.value, spec) if want_spectrum else (dt.value, var.value)

    def set_shard(self, rank, world):
        self._call("set_shard", [C.c_int, C.c_int], int(rank), int(world))

    def set_comm(self, comm):
        """Attach the library-owned NCCL communicator (Comm): sets the residual shard to its (rank, world) and routes every cross-rank
        sum through ncclAllReduce on the solver's stream.  None detaches."""
        self._call("set_comm", [C.c_void_p], comm.c if comm is not None else None)
        self._keepalive.append(comm)

    def set_allreduce(self, pyfunc):
        cb = ALLREDUCE_FN(pyfunc) if pyfunc is not None else C.cast(None, ALLREDUCE_FN)
        self._keepalive.append(cb)
        self._call("set_allreduce", [ALLREDUCE_FN, C.c_void_p], cb, None)

    def batch_init_spline(self, T_i_c_init, dt_so3_s, dt_r3_s, std_so3, std_r3, time_offset_imu_to_cam_s, init_line_delay_s,
                          acc_intrinsics=(0, 0, 0, 1, 1, 1), gyr_intrinsics=(0, 0, 0, 0, 0, 0, 1, 1, 1), acc_bias=(0, 0, 0),
                          gyr_bias=(0, 0, 0), dispatch_fov=False):
        p = InitParams()
        p.T_i_c_init[:] = list(map(float, T_i_c_init)); p.dt_so3_s = dt_so3_s; p.dt_r3_s = dt_r3_s; p.std_so3 = std_so3; p.std_r3 = std_r3
        p.time_offset_imu_to_cam_s = time_offset_imu_to_cam_s; p.init_line_delay_s = init_line_delay_s
        p.acc_intrinsics[:] = list(map(float, acc_intrinsics)); p.gyr_intrinsics[:] = list(map(float, gyr_intrinsics))
        p.acc_bias[:] = list(map(float, acc_bias)); p.gyr_bias[:] = list(map(float, gyr_bias)); p.dispatch_fov = int(bool(dispatch_fov))
        self._call("batch_init_spline", [C.POINTER(InitParams)], C.byref(p))

    def set_known_gravity_dir(self, g):
        g = _f64(g)
        self._call("set_known_gravity_dir", [c_double_p], _dp(g))

    # ---- solve ---------------------------------------------------------------------------------------------
    def optimize(self, max_iterations, flags) -> Summary:
        s = Summary()
        self._call("optimize", [C.c_int, C.c_int, C.POINTER(Summary)], int(max_iterations), int(flags), C.byref(s))
        return s

    def lm_iterations(self, n, flags) -> Summary:
        s = Summary()
        self._call("lm_iterations", [C.c_int, C.c_int, C.POINTER(Summary)], int(n), int(flags), C.byref(s))
        return s

    def time_evaluations(self, n, flags, with_jacobian=True) -> float:
        ms = C.c_double()
        self._call("time_evaluations", [C.c_int, C.c_int, C.c_int, c_double_p], int(n), int(flags), int(with_jacobian), C.byref(ms))
        return ms.value

    # ---- getters -------------------------------------------------------------------------------------------
    def get_T_i_c(self):
        T = np.zeros(7); self._call("get_T_i_c", [c_double_p], _dp(T)); return T

    def set_T_i_c(self, T):
        T = _f64(T); self._call("set_T_i_c", [c_double_p], _dp(T))

    def get_gravity(self):
        g = np.zeros(3); self._call("get_gravity", [c_double_p], _dp(g)); return g

    def get_line_delay(self):
        v = C.c_double(); self._call("get_line_delay", [c_double_p], C.byref(v)); return v.value

    def get_camera_intrinsics(self, n=10):
        k = np.zeros(n); self._call("get_camera_intrinsics", [c_double_p, C.c_int], _dp(k), n); return k

    def get_time_offset(self):
        v = C.c_double(); self._call("get_time_offset", [c_double_p], C.byref(v)); return v.value

    def set_line_delay(self, v):
        self._call("set_line_delay", [C.c_double], float(v))

    def num_knots(self):
        a, b, c, d = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        self._call("get_num_knots", [C.POINTER(C.c_int)] * 4, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return a.value, b.value, c.value, d.value

    def get_knots(self):
        a, b, c, d = self.num_knots()
        so3, r3, ba, bg = np.zeros((a, 4)), np.zeros((b, 3)), np.zeros((c, 3)), np.zeros((d, 3))
        self._call("get_knots", [c_double_p] * 4, _dp(so3), _dp(r3), _dp(ba), _dp(bg))
        return so3, r3, ba, bg

    def set_knots(self, so3=None, r3=None, ba=None, bg=None):
        arrs = [None if x is None else _f64(x) for x in (so3, r3, ba, bg)]
        self._call("set_knots", [c_double_p] * 4, *[_dp(x) for x in arrs])

    def mean_reprojection_error(self):
        v = C.c_double(); self._call("get_mean_reprojection_error", [c_double_p], C.byref(v)); return v.value

    def corner_status(self):
        """Per corner given to set_frames: 1 in this shard's solve, 0 rejected by reject_outlier_corners, -1 not assembled here."""
        st = np.zeros(self._n_corners_in, dtype=np.int32)
        self._call("get_corner_status", [C.c_int, c_int32_p], st.size, st.ctypes.data_as(c_int32_p))
        return st

    def corner_errors(self):
        """|(rx, ry)| of every corner in this shard's solve at the current state, in frame order."""
        n = int(np.count_nonzero(self.corner_status() == 1))
        e = np.zeros(n)
        self._call("get_corner_errors", [C.c_int, c_double_p], n, _dp(e))
        return e

    def reject_outlier_corners(self, k_sigma, min_px=1.0) -> dict:
        """Remove from the solve every corner whose error exceeds max(min_px, k_sigma * rms) (failed projections always)."""
        o = OutlierSummary()
        self._call("reject_outlier_corners", [C.c_double, C.c_double, C.POINTER(OutlierSummary)], float(k_sigma), float(min_px), C.byref(o))
        return o.as_dict()

    def imu_used(self):
        n = C.c_int(); self._call("get_num_imu_used", [C.POINTER(C.c_int)], C.byref(n))
        t, a, g = np.zeros(n.value), np.zeros((n.value, 3)), np.zeros((n.value, 3))
        self._call("get_imu_used", [c_double_p] * 3, _dp(t), _dp(a), _dp(g))
        return t, a, g

    def imu_cells(self):
        """Knot-interval cells of the kept IMU samples: rows (s_so3, s_r3, s_acc_bias, s_gyr_bias, i_begin, i_end)."""
        n = C.c_int(); self._call("get_num_imu_cells", [C.POINTER(C.c_int)], C.byref(n))
        c = np.zeros((n.value, 6), dtype=np.int32)
        self._call("get_imu_cells", [c_int32_p], c.ctypes.data_as(c_int32_p))
        return c

    def eval_schedule(self):
        """Per-warp runs of the persistent Jacobian kernel: dict with n_vchunks, n_ichunks and the vision / IMU runs as int32 rows
        (first unit, pos_begin, pos_end) of the packed corner / sample streams."""
        n = np.zeros(4, dtype=np.int32)
        self._call("get_eval_schedule", [c_int32_p] * 3, n.ctypes.data_as(c_int32_p), None, None)
        v, i = np.zeros((n[2], 3), dtype=np.int32), np.zeros((n[3], 3), dtype=np.int32)
        self._call("get_eval_schedule", [c_int32_p] * 3, n.ctypes.data_as(c_int32_p), v.ctypes.data_as(c_int32_p), i.ctypes.data_as(c_int32_p))
        return {"n_vchunks": int(n[0]), "n_ichunks": int(n[1]), "vitems": v, "iitems": i}

    def eval_trajectory(self, t_ns):
        t = np.ascontiguousarray(t_ns, dtype=np.int64); n = t.size
        out = dict(gyro=np.zeros((n, 3)), accel=np.zeros((n, 3)), gyro_bias=np.zeros((n, 3)), accel_bias=np.zeros((n, 3)),
                   pose_q=np.zeros((n, 4)), pose_p=np.zeros((n, 3)), valid=np.zeros(n, dtype=np.int32))
        self._call("eval_trajectory", [C.c_int, c_int64_p] + [c_double_p] * 6 + [c_int32_p], n, t.ctypes.data_as(c_int64_p), _dp(out["gyro"]),
                   _dp(out["accel"]), _dp(out["gyro_bias"]), _dp(out["accel_bias"]), _dp(out["pose_q"]), _dp(out["pose_p"]),
                   out["valid"].ctypes.data_as(c_int32_p))
        return out

    def get_stream(self) -> int:
        f = self._fn("get_stream"); f.restype = C.c_void_p; f.argtypes = [C.c_void_p]
        return int(f(self.h) or 0)

    # ---- test / measurement surface --------------------------------------------------------------------------
    def num_residuals(self):
        v, a, g = C.c_int(), C.c_int(), C.c_int()
        self._call("num_residuals", [C.POINTER(C.c_int)] * 3, C.byref(v), C.byref(a), C.byref(g))
        return v.value, a.value, g.value

    def num_tangent(self, flags):
        n = C.c_int(); self._call("num_tangent", [C.c_int, C.POINTER(C.c_int)], int(flags), C.byref(n)); return n.value

    def set_bias_splines(self, acc_dt_s=0.0, gyr_dt_s=0.0):
        """Knot spacing [s] of the accelerometer / gyroscope bias splines for the next batch_init_spline (<= 0: the reference's 10 s)."""
        self._call("set_bias_splines", [C.c_double, C.c_double], float(acc_dt_s), float(gyr_dt_s))

    def set_bias_random_walk(self, acc_q=None, gyr_q=None):
        """Random-walk densities per axis (Kalibr's units: m/s^3/sqrt(Hz), rad/s^2/sqrt(Hz)) of the bias prior for the next
        batch_init_spline; None turns that sensor's prior off."""
        arrs = [None if q is None else _f64(np.broadcast_to(np.asarray(q, dtype=np.float64), (3,))) for q in (acc_q, gyr_q)]
        self._call("set_bias_random_walk", [c_double_p, c_double_p], *[_dp(x) for x in arrs])

    def num_bias_prior_residuals(self) -> int:
        """Rows of the bias random-walk prior in this shard's problem (they follow the gyroscope rows of evaluate's residuals)."""
        n = C.c_int(); self._call("num_bias_prior_residuals", [C.POINTER(C.c_int)], C.byref(n)); return n.value

    def evaluate(self, flags, residuals=True, gradient=True, hessian=False):
        nres = sum(self.num_residuals()) + (self.num_bias_prior_residuals() if hasattr(self.lib, self.prefix + "num_bias_prior_residuals") else 0)
        n = self.num_tangent(flags)
        cost = C.c_double()
        r = np.zeros(nres) if residuals else None
        g = np.zeros(n) if gradient else None
        H = np.zeros((n, n)) if hessian else None
        self._call("evaluate", [C.c_int, c_double_p, c_double_p, c_double_p, c_double_p], int(flags), C.byref(cost), _dp(r), _dp(g), _dp(H))
        return cost.value, r, g, H


def _normal_matvec(self, flags, V):
    """J^T J V from the packed normal equations of the current state (V: (nvec, n_tangent), canonical order)."""
    V = np.ascontiguousarray(V, dtype=np.float64)
    out = np.zeros_like(V)
    self._call("normal_matvec", [C.c_int, C.c_int, c_double_p, c_double_p], int(flags), int(V.shape[0]), _dp(V), _dp(out))
    return out


CApi.normal_matvec = _normal_matvec


class SolverPlan(C.Structure):
    """icc_solver_plan_info (include/icc_b200.h): the elimination plan of the damped normal-equation solve."""
    _fields_ = [("valid", C.c_int32), ("nk", C.c_int32), ("kd", C.c_int32), ("nb", C.c_int32), ("P", C.c_int32), ("len", C.c_int32),
                ("rem", C.c_int32), ("L", C.c_int32), ("cl_global", C.c_int32), ("cs_global", C.c_int32), ("stage0", C.c_int32),
                ("WS_A", C.c_int32), ("backsub0_staged", C.c_int32), ("max_leaf", C.c_int32), ("S", C.c_int32 * 16),
                ("smem_bytes", C.c_int64 * 5), ("workspace_doubles", C.c_int64)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["S"] = list(self.S)[1:self.L + 2]
        d["smem_bytes"] = list(self.smem_bytes)
        return d


def _solver_plan(self, flags, chunks=0) -> dict:
    """The plan the solve would use under `flags` with `chunks` level-0 chunks (0 = the planner's choice); host only."""
    p = SolverPlan()
    self._call("solver_plan", [C.c_int, C.c_int, C.POINTER(SolverPlan)], int(flags), int(chunks), C.byref(p))
    return p.as_dict()


def _solve_normal_equations(self, flags, radius, chunks=0) -> dict:
    """One damped solve of the normal equations left by the preceding evaluate / normal_matvec with the same flags
    -> dict(delta, scale, h_diag, model_change, step_ok, plan), vectors in canonical tangent order."""
    n = self.num_tangent(flags)
    d, s, hd = np.full(n, np.nan), np.zeros(n), np.zeros(n)
    mc, ok, p = C.c_double(), C.c_int32(), SolverPlan()
    self._call("solve_normal_equations", [C.c_int, C.c_double, C.c_int, c_double_p, c_double_p, c_double_p, c_double_p, c_int32_p, C.POINTER(SolverPlan)],
               int(flags), float(radius), int(chunks), _dp(d), _dp(s), _dp(hd), C.byref(mc), C.byref(ok), C.byref(p))
    return dict(delta=d, scale=s, h_diag=hd, model_change=mc.value, step_ok=ok.value, plan=p.as_dict())


def kernel_launch_count(lib) -> int:
    """CUDA kernels the library has launched in this process (all handles)."""
    f = lib.icc_kernel_launch_count; f.restype = C.c_int64; f.argtypes = []
    return int(f())


CApi.solver_plan = _solver_plan
CApi.solve_normal_equations = _solve_normal_equations


class Comm:
    """icc_comm: the library's own NCCL communicator (include/icc_b200.h).  `unique_id()` on one rank, `Comm(lib, id, rank, world,
    device)` on every rank (collective)."""
    ID_BYTES = 128

    @staticmethod
    def unique_id(lib) -> bytes:
        buf = (C.c_ubyte * Comm.ID_BYTES)()
        f = lib.icc_comm_unique_id; f.restype = C.c_int; f.argtypes = [C.c_void_p]
        st = f(buf)
        if st != 0:
            e = lib.icc_comm_last_error; e.restype = C.c_char_p
            raise IccError(f"icc_comm_unique_id: {STATUS_NAMES.get(st, st)}: {(e() or b'').decode()}")
        return bytes(buf)

    def __init__(self, lib, uid: bytes, rank: int, world: int, device: int):
        self.lib, self.rank, self.world = lib, int(rank), int(world)
        out = C.c_void_p()
        buf = (C.c_ubyte * Comm.ID_BYTES).from_buffer_copy(uid)
        f = lib.icc_comm_create; f.restype = C.c_int; f.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_int, C.c_int]
        st = f(C.byref(out), buf, int(rank), int(world), int(device))
        if st != 0:
            e = lib.icc_comm_last_error; e.restype = C.c_char_p
            raise IccError(f"icc_comm_create: {STATUS_NAMES.get(st, st)}: {(e() or b'').decode()}")
        self.c = out

    def close(self):
        if getattr(self, "c", None):
            f = self.lib.icc_comm_destroy; f.restype = None; f.argtypes = [C.c_void_p]
            f(self.c); self.c = None


def default_solver_options() -> SolverOptions:
    """ceres::Solver::Options of SplineTrajectoryEstimator::Optimize (impl.h:254-266) + Ceres 2.1 defaults."""
    return SolverOptions(1e-4, 1e-7, 1e-10, 1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 1, 5)


def load_dataset(api: CApi, ds: dict, known_gravity=True, dispatch_fov=None, shard=None, comm=None):
    """Feed a synthetic dataset (synthetic.make_dataset) through the boundary in the order the hot CLI does."""
    W, H = ds["image_size"]
    api.set_camera(ds["model"], ds["intrinsics"], W, H)
    api.set_board_points(ds["board_xyzw"])
    api.set_frames(ds["frame_t"], ds["corner_offsets"], ds["point_ids"], ds["uv"], ds["q_wc"], ds["p_wc"])
    api.set_imu(ds["imu_t"], ds["accel"], ds["gyro"])
    if shard is not None:
        api.set_shard(*shard)
    if comm is not None:
        api.set_comm(comm)
    if dispatch_fov is None:
        dispatch_fov = ds["model"] == 3
    api.batch_init_spline(ds["T_i_c_init"], ds["dt_so3_s"], ds["dt_r3_s"], ds["std_so3"], ds["std_r3"], ds["time_offset_imu_to_cam_s"],
                          ds["init_line_delay_s"], acc_bias=ds["acc_bias"], gyr_bias=ds["gyr_bias"], dispatch_fov=dispatch_fov)
    if known_gravity:
        api.set_known_gravity_dir(ds["gravity"])
