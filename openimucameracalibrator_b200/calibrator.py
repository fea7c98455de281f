"""Python host mirror of OpenICC::core::ImuCameraCalibrator (include/OpenCameraCalibrator/core/imu_camera_calibrator.h:29-118)
on top of the CUDA C-ABI.  Same method names, argument meaning and error behaviour; there is no CPU fallback — a missing
`libicc_b200.so` or a missing GPU raises."""
from __future__ import annotations

import ctypes
import enum
import os

import numpy as np

from . import _capi
from ._capi import CApi, IccError

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def library_path() -> str:
    return os.path.join(_HERE, "libicc_b200.so")


def load_library() -> ctypes.CDLL:
    """Load the in-tree CUDA library; fails loudly when it has not been built (`python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _LIB
    if _LIB is None:
        path = library_path()
        if not os.path.exists(path):
            raise IccError(f"{path} is missing: build the CUDA extension first (__graft_entry__.build()); there is no CPU fallback")
        _LIB = ctypes.CDLL(path)
    return _LIB


class SplineOptimFlags(enum.IntFlag):
    """core/spline_trajectory_estimator.h:17-27"""
    POINTS = 1
    T_I_C = 2
    IMU_BIASES = 4
    IMU_INTRINSICS = 8
    GRAVITY_DIR = 16
    CAM_LINE_DELAY = 32
    SPLINE = 64
    ACC_BIAS = 128
    GYR_BIAS = 256


class ImuCameraCalibrator:
    """`BatchInitSpline` -> `Optimize` -> getters, as driven by continuous_time_imu_to_camera_calibration.cc:191-263."""

    def __init__(self, device: int = 0):
        self.api = CApi(load_library(), "icc_", int(device))
        self._cam_timestamps = None

    # -- problem data (what main() assembles into theia::Reconstruction / CameraTelemetryData) --------------------
    def SetCamera(self, model: int, intrinsics, image_width: int, image_height: int):
        self.api.set_camera(model, intrinsics, image_width, image_height)

    def SetBoardPoints(self, xyzw):
        self.api.set_board_points(xyzw)

    def SetViews(self, timestamps_s, corner_offsets, point_ids, uv, q_wc_xyzw, p_wc):
        self._cam_timestamps = np.sort(np.asarray(timestamps_s, dtype=np.float64))
        self.api.set_frames(timestamps_s, corner_offsets, point_ids, uv, q_wc_xyzw, p_wc)

    def SetTelemetry(self, timestamps_s, accelerometer, gyroscope):
        self.api.set_imu(timestamps_s, accelerometer, gyroscope)

    def SetShard(self, rank: int, world: int):
        self.api.set_shard(rank, world)

    def SetReprojectionError(self, mode: str):
        """"pixel" (default, the reference's residual) or "tangent" (corners as unit bearings); before BatchInitSpline."""
        self.api.set_reprojection_error(mode)

    # -- reference API ------------------------------------------------------------------------------------------------
    def BatchInitSpline(self, T_i_c_init, dt_so3, dt_r3, std_so3, std_r3, time_offset_imu_to_cam, initial_line_delay,
                        accl_intrinsics=(0, 0, 0, 1, 1, 1), gyro_intrinsics=(0, 0, 0, 0, 0, 0, 1, 1, 1), accl_bias=(0, 0, 0),
                        gyro_bias=(0, 0, 0), dispatch_fov=False):
        self.api.batch_init_spline(T_i_c_init, dt_so3, dt_r3, std_so3, std_r3, time_offset_imu_to_cam, initial_line_delay,
                                   accl_intrinsics, gyro_intrinsics, accl_bias, gyro_bias, dispatch_fov)

    def SetKnownGravityDir(self, gravity):
        self.api.set_known_gravity_dir(gravity)

    def Optimize(self, iterations: int, optim_flags: int) -> float:
        """Returns the mean reprojection error like the reference (imu_camera_calibrator.cc:163-168)."""
        self.last_summary = self.api.optimize(iterations, int(optim_flags))
        return self.last_summary.mean_reproj_error

    def SetBiasSplines(self, acc_dt_s: float, gyr_dt_s: float):
        """Bias-spline knot spacing [s] for the next BatchInitSpline (<= 0: the reference's 10 s)."""
        self.api.set_bias_splines(acc_dt_s, gyr_dt_s)

    def SetBiasRandomWalk(self, acc_q, gyr_q):
        """Random-walk prior on the bias splines for the next BatchInitSpline: per-axis densities in Kalibr's units (scalar or 3-vector,
        m/s^3/sqrt(Hz) and rad/s^2/sqrt(Hz); io_formats.bias_random_walk_from_allan derives them from an Allan fit); None: no prior."""
        self.api.set_bias_random_walk(acc_q, gyr_q)

    def GetCornerErrors(self):
        """Per-corner reprojection error |(rx, ry)| [px, or scaled tangent units] of the corners in the solve, in frame order."""
        return self.api.corner_errors()

    def RejectOutlierCorners(self, k_sigma: float, min_px: float = 1.0) -> dict:
        """Drop the corners whose error exceeds max(min_px, k_sigma * rms) until the next BatchInitSpline (icc_reject_outlier_corners)."""
        return self.api.reject_outlier_corners(k_sigma, min_px)

    def GetCornerStatus(self):
        """Per input corner: 1 in the solve, 0 rejected, -1 not assembled (icc_get_corner_status)."""
        return self.api.corner_status()

    def GetCamTimestamps(self):
        return self._cam_timestamps

    def GetGyroMeasurements(self):
        t, _, g = self.api.imu_used()
        return t, g

    def GetAcclMeasurements(self):
        t, a, _ = self.api.imu_used()
        return t, a

    def GetCalibratedRSLineDelay(self) -> float:
        return self.api.get_line_delay()

    def GetT_i_c(self):
        return self.api.get_T_i_c()

    def GetGravity(self):
        return self.api.get_gravity()

    def EvalTrajectory(self, t_ns):
        """GetAngularVelocity / GetAcceleration / GetGyroBias / GetAcclBias / GetPose for many timestamps at once."""
        return self.api.eval_trajectory(t_ns)

    @classmethod
    def from_dataset(cls, ds: dict, device: int = 0, known_gravity: bool = True, shard=None) -> "ImuCameraCalibrator":
        self = cls(device)
        _capi.load_dataset(self.api, ds, known_gravity=known_gravity, shard=shard)
        self._cam_timestamps = np.sort(np.asarray(ds["frame_t"], dtype=np.float64))
        return self


class CameraCalibrator:
    """Python host mirror of OpenICC::core::CameraCalibrator (include/OpenCameraCalibrator/core/camera_calibrator.h:25-86,
    SURVEY.md §8(f) row f4): `CalibrateCameraFromJson` (src/core/camera_calibrator.cc:221-389) with the corner-file dictionary the
    reference's tools exchange, or `AddView` / `AddObservation` / `RunCalibration` (:78-219) with caller-made initial poses.  The
    bundle adjustment runs on the GPU behind `icc_calibrate_camera`; there is no CPU fallback."""

    def __init__(self, camera_model: str, optimize_board_pts: bool = False, device: int = 0):
        from . import camera_models as cm
        if camera_model not in cm.MODEL_IDS:
            raise IccError(f"unknown camera model {camera_model!r}")
        self.camera_model, self.model = camera_model, cm.MODEL_IDS[camera_model]
        self.optimize_board_pts = bool(optimize_board_pts)        # camera_calibrator.cc:207-216; refined points: self.api.get_board_points()
        self.api = CApi(load_library(), "icc_", int(device))
        self.grid_size, self.verbose = 0.04, False
        self._views, self._obs = [], {}
        self._image_size = None
        self._rolling, self._line_delay = False, 0.0
        self.result = None

    def SetGridSize(self, grid_size: float = 0.04):
        self.grid_size = float(grid_size)

    def SetVerbose(self):
        self.verbose = True

    def SetRollingShutter(self, line_delay_s=None):
        """Rolling-shutter calibration (icc_set_camcal_rolling_shutter, automatic mode) with the view timestamps this object holds: the
        AddView times, or the corner file's view times.  line_delay_s None takes one readout per frame interval from the corner file,
        1 / camera_fps / image_height (CalibrateCameraFromJson only); 0 returns to the global shutter."""
        if line_delay_s is None:
            self._rolling, self._line_delay = True, None
            return
        ld = float(line_delay_s)
        if not np.isfinite(ld) or ld < 0.0:
            raise IccError(f"line delay must be finite and >= 0, not {line_delay_s!r}")
        self._rolling, self._line_delay = ld > 0.0, ld

    def _set_shutter(self, times_s, line_delay_s):
        self.api.set_camcal_rolling_shutter(line_delay_s if self._rolling else 0.0, frame_t_s=times_s if self._rolling else None)

    def SetBoardPoints(self, xyzw):
        self.api.set_board_points(xyzw)

    def AddView(self, initial_rotation, initial_position, initial_focal_length, initial_distortion, image_width, image_height, timestamp_s, group_id=0):
        """initial_rotation = R_cw (theia::Camera::SetOrientationFromRotationMatrix), initial_position = camera centre in the world."""
        from .synthetic import matrix_to_quat_xyzw
        R = np.asarray(initial_rotation, dtype=np.float64).reshape(3, 3)
        self._views.append(dict(q_wc=matrix_to_quat_xyzw(R.T[None])[0], p_wc=np.asarray(initial_position, dtype=np.float64), f=float(initial_focal_length),
                                k=float(initial_distortion), t=float(timestamp_s)))
        self._image_size = (int(image_width), int(image_height))
        self._obs[len(self._views) - 1] = []
        return len(self._views) - 1

    def AddObservation(self, view_id, object_point_id, corner) -> bool:
        if view_id not in self._obs:
            return False
        self._obs[view_id].append((int(object_point_id), float(corner[0]), float(corner[1])))
        return True

    def RunCalibration(self) -> bool:
        """Three-stage bundle adjustment from the views added so far (all of them: the grid filter belongs to CalibrateCameraFromJson)."""
        if not self._views:
            return False
        off, ids, uv = [0], [], []
        for v in range(len(self._views)):
            for pid, x, y in self._obs[v]:
                ids.append(pid); uv.append((x, y))
            off.append(len(ids))
        last = self._views[-1]                                     # the shared intrinsics keep the values of the last AddView (:101-113)
        W, H = self._image_size
        if self._rolling and self._line_delay is None:
            raise IccError("RunCalibration needs SetRollingShutter(line_delay_s) with a number")
        self._set_shutter([v["t"] for v in self._views], self._line_delay)
        self.result = self.api.calibrate_camera(self.model, W, H, off, ids, np.array(uv).reshape(-1, 2), q_wc_init=np.array([v["q_wc"] for v in self._views]),
                                                p_wc_init=np.array([v["p_wc"] for v in self._views]), focal_length_init=last["f"], distortion_init=last["k"], grid_size=0.0,
                                                optimize_board_points=int(self.optimize_board_pts))
        return bool(self.result["summary"]["success"])

    def CalibrateCameraFromJson(self, scene_json: dict, output_path: str = "") -> bool:
        """scene_json: the corner file as a dictionary (io_formats.ubjson_loads of extract_board_to_json's output).  Writes
        `<output_path>.json` in the layout of io::write_camera_calibration when output_path is given."""
        import json
        from .io_formats import intrinsics_dict
        pts = scene_json["scene_pts"]
        if isinstance(pts, (list, tuple)):                         # the reference's radon files: an array indexed by id
            pts = {i: p for i, p in enumerate(pts)}
        n = max(int(i) for i in pts) + 1
        board = np.zeros((n, 4)); board[:, 3] = 1.0
        for i, p in pts.items():
            board[int(i), :3] = p
        self.api.set_board_points(board)
        W, H = int(scene_json["image_width"]), int(scene_json["image_height"])
        off, ids, uv, self._timestamps_s = [0], [], [], []
        for key in sorted(scene_json["views"]):                    # nlohmann::json objects iterate in key order
            ip = scene_json["views"][key]["image_points"]
            for pid in sorted(ip):
                ids.append(int(pid)); uv.append(ip[pid])
            off.append(len(ids)); self._timestamps_s.append(float(key) * 1e-6)
        if self._rolling and self._line_delay is None:
            fps = float(scene_json["camera_fps"])
            if not (fps > 0.0 and H > 0):
                raise IccError("a rolling shutter needs camera_fps > 0 and image_height > 0 in the corner file")
            self._set_shutter(self._timestamps_s, 1.0 / fps / H)
        else:
            self._set_shutter(self._timestamps_s, self._line_delay)
        self.result = self.api.calibrate_camera(self.model, W, H, off, ids, np.array(uv, dtype=np.float64).reshape(-1, 2), grid_size=self.grid_size,
                                                optimize_board_points=int(self.optimize_board_pts))
        s = self.result["summary"]
        if not s["success"]:
            return False
        if output_path:
            doc = {"stabelized": False, "fps": scene_json["camera_fps"], "nr_calib_images": s["n_views_used"], "final_reproj_error": s["final_reproj_error"],
                   "image_width": W, "image_height": H, "intrinsic_type": self.camera_model, "intrinsics": intrinsics_dict(self.model, self.result["intrinsics"])}
            with open(output_path + ".json", "w") as f:
                json.dump(doc, f, indent=2)
        return True

    def PrintResult(self):
        from . import camera_models as cm
        k = self.result["intrinsics"]
        cam = cm.CAMERAS[self.model]
        print(f"Focal Length:{k[0]}px Principal Point: {k[cam.keys['principal_pt_x']]}/{k[cam.keys['principal_pt_y']]}px.")
        if cam.printed:
            print(f"{cam.name} model: " + " ".join(f"{label}: {k[i]}" if label else f"{k[i]}" for label, i in cam.printed.items()))


class StaticImuCalibrator:
    """OpenICC::core::StaticImuCalibrator (include/OpenCameraCalibrator/core/static_imu_calibrator.h) on the CUDA C-ABI: the same
    setters and getters; CalibrateAccGyro runs icc_static_imu_calibration.  Calibrations are returned as parameter vectors
    (acc [misYZ, misZY, misZX, sX, sY, sZ, bX, bY, bZ]; gyro [misYZ, misZY, misZX, misXZ, misXY, misYX, sX, sY, sZ] + bias)."""

    def __init__(self, device: int = 0):
        self._api = CApi(load_library(), "icc_", device)
        self._opt = {}
        self._acc = np.array([0, 0, 0, 1, 1, 1, 0, 0, 0], dtype=float)
        self._gyr = np.array([0, 0, 0, 0, 0, 0, 1, 1, 1], dtype=float)
        self._gyr_bias = np.zeros(3)
        self.summary = None

    def SetGravityMagnitude(self, g: float):
        self._opt["g_mag"] = g

    def SetInitStaticIntervalDuration(self, duration_s: float):
        self._opt["init_interval_duration_s"] = duration_s

    def SetIntarvalsNumSamples(self, num: int):
        self._opt["interval_n_samples"] = num

    def SetInitAccCalibration(self, mis_scale6):
        self._opt["init_acc"] = list(mis_scale6)

    def SetInitGyroCalibration(self, mis_scale9):
        self._opt["init_gyr"] = list(mis_scale9)

    def EnableAccUseMeans(self, enabled: bool):
        self._opt["acc_use_means"] = int(bool(enabled))

    def SetGyroDataPeriod(self, dt: float):
        self._opt["gyro_dt"] = dt

    def EnableGyroBiasOptimization(self, enabled: bool):
        self._opt["optimize_gyro_bias"] = int(bool(enabled))

    def CalibrateAccGyro(self, timestamps_s, accelerometer, gyroscope) -> bool:
        r = self._api.static_imu_calibration(timestamps_s, accelerometer, gyroscope, **self._opt)
        self._acc, self._gyr, self._gyr_bias, self.summary = r["acc_params"], r["gyr_params"], r["gyr_bias"], r["summary"]
        return bool(self.summary["success"])

    def getAccCalib(self):
        return self._acc.copy()

    def getGyroCalib(self):
        """-> (gyr_params[9], bias[3])"""
        return self._gyr.copy(), self._gyr_bias.copy()


class AllanVarianceFitter:
    """OpenICC::core::AllanVarianceFitter (include/OpenCameraCalibrator/core/allan_variance_fitter.h) on the CUDA C-ABI: constructed from
    the telemetry (timestamps [s], accelerometer [m/s^2] and gyroscope [rad/s] as (n, 3)) and the number of clusters; RunFit runs
    icc_allan_variance.  Afterwards `params` (6, 5) holds [Q, N, B, K, R] per channel (acc x, y, z, gyr x, y, z), `noise` and `summary`
    the derived quantities and fit statistics per channel, and curves(c) the sigma^2 curve and its fit."""

    def __init__(self, timestamps_s, accelerometer, gyroscope, nr_clusters: int = 10000, device: int = 0):
        self._api = CApi(load_library(), "icc_", device)
        self._data = (timestamps_s, accelerometer, gyroscope)
        self.nr_clusters = nr_clusters
        self.params = self.noise = self.summary = None

    def RunFit(self) -> bool:
        r = self._api.allan_variance(*self._data, n_clusters=self.nr_clusters)
        self.params, self.noise, self.summary = r["params"], r["noise"], r["summary"]
        return True

    def curves(self, channel: int) -> dict:
        return self._api.allan_curves(channel)


class BoardExtractor:
    """BoardExtractor for BoardType::RADON (src/core/board_extractor.cc) on the GPU: InitializeRadonBoard, then frames -> the scene
    dictionary of the corner file (the layout io_formats.write_dataset_files writes and icccli::load_scene reads)."""

    def __init__(self, square_length_m: float, corners_x: int = 14, corners_y: int = 9, device: int = 0):
        self.square_length_m, self.corners_x, self.corners_y = float(square_length_m), int(corners_x), int(corners_y)
        self.api = CApi(load_library(), "icc_", device)

    def scene_points(self) -> dict:
        """id -> (i s, j s, 0): the reference puts the row index i on x (InitializeRadonBoard)."""
        s, W = self.square_length_m, self.corners_x
        return {str(i * W + j): [float(i * s), float(j * s), 0.0] for i in range(self.corners_y) for j in range(W)}

    def extract(self, frames, timestamps_s, downsample_factor: float = 1.0) -> dict:
        """Corner-file dictionary of the frames: views named io_formats.view_key(t), written only for frames where the board was found."""
        from .io_formats import view_key
        uv, found, summary = self.api.extract_radon_board(frames, self.corners_x, self.corners_y, downsample_factor)
        views = {}
        for k, t in enumerate(timestamps_s):
            if found[k]:
                views[view_key(float(t))] = {"image_points": {str(c): [float(uv[k, c, 0]), float(uv[k, c, 1])] for c in range(uv.shape[1])}}
        self.summary = summary
        return {"calibration_board_type": 1, "square_size_meter": self.square_length_m, "image_width": int(summary["width"]),
                "image_height": int(summary["height"]), "scene_pts": self.scene_points(), "views": views}

    def write(self, path: str, frames, timestamps_s, downsample_factor: float = 1.0) -> dict:
        """extract(), written as UBJSON with io_formats.ubjson_dumps; returns the dictionary."""
        from .io_formats import ubjson_dumps
        scene = self.extract(frames, timestamps_s, downsample_factor)
        with open(path, "wb") as f:
            f.write(ubjson_dumps(scene))
        return scene


class AprilGridExtractor(BoardExtractor):
    """BoardExtractor for BoardType::APRILTAG (src/core/board_extractor.cc) on the GPU: InitializeAprilBoard(tag_size_m, 0.3, tags_x,
    tags_y), then frames -> the corner file's scene dictionary.  A view holds only the kept corners (status 1) of its frame; frames
    without a view (fewer than 4 tags, or a duplicate id) are left out.  write() is BoardExtractor's."""

    def __init__(self, tag_size_m: float, tags_x: int = 6, tags_y: int = 6, device: int = 0):
        self.tag_size_m, self.tags_x, self.tags_y = float(tag_size_m), int(tags_x), int(tags_y)
        self.api = CApi(load_library(), "icc_", device)

    def scene_points(self) -> dict:
        """str((t << 2) + i) -> the corner as cv::Point3f: tag t = tags_x y + x, corner i at (1.3 s x + {0, s, s, 0}[i],
        1.3 s y + {0, 0, s, s}[i], 0), each coordinate rounded to float32 as the reference stores it."""
        import numpy as np
        s, nx = self.tag_size_m, self.tags_x
        out = {}
        for t in range(nx * self.tags_y):
            x, y = t % nx, t // nx
            for i in range(4):
                p = np.array([x * s * 1.3 + (0.0, s, s, 0.0)[i], y * s * 1.3 + (0.0, 0.0, s, s)[i], 0.0], dtype=np.float32)
                out[str((t << 2) + i)] = [float(v) for v in p]
        return out

    def extract(self, frames, timestamps_s, downsample_factor: float = 1.0) -> dict:
        import numpy as np
        from .io_formats import view_key
        uv, status, found, summary = self.api.extract_aprilgrid(frames, self.tags_x, self.tags_y, downsample_factor)
        views = {}
        for k, t in enumerate(timestamps_s):
            if found[k]:
                ids = [int(c) for c in range(status.shape[1]) if status[k, c] == 1]
                views[view_key(float(t))] = {"image_points": {str(c): [float(uv[k, c, 0]), float(uv[k, c, 1])] for c in ids}}
        self.summary = summary
        scene = {"calibration_board_type": 2, "square_size_meter": self.tag_size_m, "image_width": int(summary["width"]),
                 "image_height": int(summary["height"]), "scene_pts": self.scene_points(), "views": views}
        t = np.asarray(timestamps_s, dtype=np.float64)
        if t.size >= 3:   # the reference's camera_fps: 1 / the median frame interval, the last interval left out
            scene["camera_fps"] = float(1.0 / np.median(np.diff(t)[:-1]))
        return scene
