// Drop-in host program for applications/estimate_imu_to_camera_rotation.cc of urbste/OpenImuCameraCalibrator (SURVEY.md §8(f)
// row f3): same gflags names (app :30-53), same telemetry / bias JSON inputs, same output JSON keys (app :175-185:
// gyro_bias, gyro_to_camera_rotation{w,x,y,z}, time_offset_gyro_to_cam) -- the file the hot CLI reads as
// --gyro_to_cam_initial_calibration.  The estimation runs on the GPU through icc_estimate_imu_to_camera_rotation
// (ImuToCameraRotationEstimator::EstimateCameraImuRotation, src/core/imu_to_camera_rotation_estimator.cc:116-274).
//
// One deliberate difference: --input_pose_calibration_dataset is the JSON pose dataset of this repository
// ({"views": {"<name>": {"q_wc": [w,x,y,z], "p_wc": [...], "timestamp_s": t}}}; without "timestamp_s" the view name, which is
// (uint64) timestamp_us, gives the time), not Theia's cereal-binary Reconstruction.  Extra flag: --device.
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"

#include <fstream>
#include <iostream>

using iccjson::Value;

int main(int argc, char** argv) {
  icccli::Flags F;
  F.str = {{"input_pose_calibration_dataset", ""}, {"telemetry_json", ""}, {"imu_bias_estimate", ""}, {"imu_rotation_init_output", "gyro_to_cam_calibration.json"}};
  F.num = {{"delta_t_imu_to_cam", 0.0}, {"device", 0.0}};
  try { icccli::parse_flags(argc, argv, F); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  try {
    Value poses;
    try { poses = iccjson::load_json(F.str["input_pose_calibration_dataset"]); }
    catch (const std::exception& e) { std::cerr << "Check failed: could not read the pose dataset (JSON expected): " << e.what() << std::endl; return 1; }
    icccli::Telemetry tel;
    try { tel = icccli::load_telemetry(F.str["telemetry_json"]); } catch (const std::exception& e) { std::cerr << "Could not read: " << F.str["telemetry_json"] << ": " << e.what() << std::endl; return 1; }
    double bias[3] = {0, 0, 0}; bool have_bias = false;
    if (!F.str["imu_bias_estimate"].empty()) {      // ReadIMUBias (src/io/read_misc.cc:49-63)
      const Value b = iccjson::load_json(F.str["imu_bias_estimate"]); const char* ax[3] = {"x", "y", "z"};
      for (int d = 0; d < 3; ++d) bias[d] = b.at("gyro_bias").at(ax[d]).num();
      have_bias = true;
    }
    if (tel.gyr.size() != 3 * tel.t_ns.size()) { std::cerr << "Telemetry should have the same amount of timestamps and gyroscope values." << std::endl; return 1; }
    std::vector<double> imu_t(tel.t_ns.size());
    for (size_t i = 0; i < imu_t.size(); ++i) imu_t[i] = tel.t_ns[i] * 1e-9;
    const std::vector<double>& gyr = tel.gyr;
    double delta_t0_cam = 0.0;                       // app :80-86
    if (!tel.img_t_ns.empty()) delta_t0_cam = tel.img_t_ns[0] * 1e-9;
    std::vector<double> view_t, q_cw;
    for (const auto& kv : *poses.at("views").o) {
      const double t = kv.second.contains("timestamp_s") ? kv.second.at("timestamp_s").num() : std::stod(kv.first) * 1e-6;
      view_t.push_back(t + delta_t0_cam);
      const Value& q = kv.second.at("q_wc");          // [w, x, y, z] of R_cw^T ; the estimator wants R_cw (app :125-127)
      q_cw.push_back(-q.at(1).num()); q_cw.push_back(-q.at(2).num()); q_cw.push_back(-q.at(3).num()); q_cw.push_back(q.at(0).num());
    }
    icc_handle* h = nullptr;
    icc_status st = icc_create(&h, (int)F.num["device"]);
    if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    double q[4], td = 0, bias_out[3], err = 0; int32_t iters = 0;
    st = icc_estimate_imu_to_camera_rotation(h, (int)view_t.size(), view_t.data(), q_cw.data(), (int)imu_t.size(), imu_t.data(), gyr.data(), have_bias ? bias : nullptr,
                                             q, &td, bias_out, &err, &iters);
    if (st != ICC_OK) { std::cerr << "rotation estimation failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    icc_destroy(h);
    std::cout << "Finished golden-section search in " << iters << " iterations.\n"
              << "Final gyro to camera quaternion is: " << q[3] << " " << q[0] << " " << q[1] << " " << q[2] << "\n"
              << "Gyro bias is estimated to be: " << bias_out[0] << ", " << bias_out[1] << ", " << bias_out[2] << "rad/s\n"
              << "Estimated time offset: " << td << "s\nFinal alignment error: " << err << "\n";
    Value out = Value::object();
    out["gyro_bias"] = Value::array(); for (int d = 0; d < 3; ++d) out["gyro_bias"].push_back(Value(bias_out[d]));
    out["gyro_to_camera_rotation"] = Value::object();
    out["gyro_to_camera_rotation"]["w"] = Value(q[3]); out["gyro_to_camera_rotation"]["x"] = Value(q[0]); out["gyro_to_camera_rotation"]["y"] = Value(q[1]); out["gyro_to_camera_rotation"]["z"] = Value(q[2]);
    out["time_offset_gyro_to_cam"] = Value(td);
    std::ofstream f(F.str["imu_rotation_init_output"]);
    if (!f.is_open()) { std::cerr << "could not write " << F.str["imu_rotation_init_output"] << std::endl; return 1; }
    f << iccjson::dump(out, 4) << std::endl;
  } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  return 0;
}
