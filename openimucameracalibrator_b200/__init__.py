"""openimucameracalibrator_b200 — H100-native (sm_90a) continuous-time IMU-camera calibration solver.

Drop-in for the one hot path of urbste/OpenImuCameraCalibrator: the spline batch optimisation behind
`applications/continuous_time_imu_to_camera_calibration.cc`.  The compute lives in `libicc_b200.so` (hand-written CUDA
behind the C-ABI of include/icc_b200.h); this package is the Python host mirror of the reference's
`OpenICC::core::ImuCameraCalibrator` interface plus the synthetic-sequence generator and file-format helpers.
"""
from .calibrator import CameraCalibrator, ImuCameraCalibrator, SplineOptimFlags, load_library, library_path  # noqa: F401

__all__ = ["CameraCalibrator", "ImuCameraCalibrator", "SplineOptimFlags", "load_library", "library_path"]
