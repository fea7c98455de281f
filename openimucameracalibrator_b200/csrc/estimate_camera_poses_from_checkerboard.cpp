// Drop-in host program for applications/estimate_camera_poses_from_checkerboard.cc of urbste/OpenImuCameraCalibrator
// (SURVEY.md §8(f) row f1): same gflags names (app :34-41), same inputs (UBJSON corner file, camera calibration JSON); every
// view's board pose is estimated on the GPU through icc_estimate_board_poses (PoseEstimator::EstimatePosesFromJson,
// src/core/pose_estimator.cc:92-191).
//
// One deliberate difference: --output_pose_dataset is written as the JSON pose dataset that this repository's
// continuous_time_imu_to_camera_calibration reads ({"views": {"<name>": {"q_wc": [w,x,y,z], "p_wc": [x,y,z], "timestamp_s": t,
// "mean_reproj_error": e}}, "tracks": {"<id>": [x,y,z,w]}}), not as Theia's cereal-binary Reconstruction (unreadable without
// Theia).  --optimize_board_points (app :61-65) runs icc_optimize_board_points (PoseEstimator::OptimizeBoardPoints + OptimizeAllPoses)
// and writes the refined board points as the dataset's tracks; PoseEstimator::FilterBadPoses (app :66-67) is applied like in the
// reference.  Extra flags: --device (CUDA ordinal, default 0); --pose_error normalized|tangent (default normalized, the reference's
// residual): tangent scores corners as unit bearings with the local tangent reprojection error, which keeps the corners and views of
// fisheye lenses beyond 90 degrees (icc_set_pose_error); the written mean_reproj_error is then in tangent units.  --pose_shutter global|rolling
// (default global): rolling reports each view's pose at its frame timestamp from corners exposed row by row, line delay 1 / fps / height
// of the camera calibration (icc_set_pose_rolling_shutter); the pose dataset keeps its format.
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"

#include <cmath>
#include <fstream>
#include <iostream>

using iccjson::Value;

int main(int argc, char** argv) {
  icccli::Flags F;
  F.str = {{"input_corners", ""}, {"camera_calibration_json", ""}, {"output_pose_dataset", ""}, {"pose_error", "normalized"}, {"pose_shutter", "global"}};
  F.boolean = {{"optimize_board_points", false}};
  F.num = {{"device", 0.0}};
  int pose_error = ICC_POSE_ERROR_NORMALIZED;
  bool rolling = false;
  try { icccli::parse_flags(argc, argv, F); pose_error = icccli::parse_pose_error(F.str["pose_error"]); rolling = icccli::parse_pose_shutter(F.str["pose_shutter"]); }
  catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  try {
    Value scene_json; icccli::SceneViews sv;
    try { scene_json = icccli::load_scene(F.str["input_corners"], sv); } catch (const std::exception& e) { std::cerr << "Check failed: Failed to load " << F.str["input_corners"] << ": " << e.what() << std::endl; return 1; }
    std::vector<double> intr; int width = 0, height = 0; double fps = 0; int model = -1;
    try { model = icccli::read_camera(iccjson::load_json(F.str["camera_calibration_json"]), intr, width, height, fps); }
    catch (const std::exception& e) { std::cerr << "Check failed: Could not read camera calibration: " << F.str["camera_calibration_json"] << ": " << e.what() << std::endl; return 1; }
    double line_delay = 0.0;
    if (rolling) { try { line_delay = icccli::pose_line_delay(fps, height); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; } }
    int np = 0;
    const std::vector<double> board = icccli::read_scene_points(scene_json, np);
    const int nv = (int)sv.timestamp_us.size();
    if (nv == 0) { std::cerr << "Check failed: the corner file holds no views" << std::endl; return 1; }
    std::cout << "PoseEstimator setting max reprojection error to: " << 0.004 * height << "\n";
    icc_handle* h = nullptr;
    icc_status st = icc_create(&h, (int)F.num["device"]);
    if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    std::vector<double> q(4 * (size_t)nv), p(3 * (size_t)nv), err(nv); std::vector<int32_t> valid(nv);
    st = icc_set_camera(h, model, intr.data(), (int)intr.size(), width, height);
    if (st == ICC_OK) st = icc_set_board_points(h, np, board.data());
    if (st == ICC_OK) st = icc_set_pose_error(h, pose_error);
    std::vector<double> frame_t(nv);
    for (int i = 0; i < nv; ++i) frame_t[i] = sv.timestamp_us[i] * 1e-6;
    if (st == ICC_OK && rolling) st = icc_set_pose_rolling_shutter(h, line_delay, nv, frame_t.data());
    if (st == ICC_OK) st = icc_estimate_board_poses(h, nv, sv.off.data(), sv.ids.data(), sv.uv.data(), 0.0, 0, q.data(), p.data(), err.data(), valid.data());
    if (st != ICC_OK) { std::cerr << "board pose estimation failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    auto report_shutter = [&]() {
      std::vector<double> vel(6 * (size_t)nv); int32_t n_static = 0;
      if (icc_get_pose_velocities(h, nv, vel.data(), &n_static) == ICC_OK)
        std::cout << "Rolling shutter: line delay " << line_delay << " s, " << n_static << " valid views without a neighbour in time keep the global-shutter model.\n";
    };
    if (rolling) report_shutter();
    std::vector<double> board_out(board);
    if (F.boolean["optimize_board_points"]) {                                  // app :61-65
      int32_t n_opt = 0;
      st = icc_optimize_board_points(h, nv, sv.off.data(), sv.ids.data(), sv.uv.data(), 0.0, 0, 0, q.data(), p.data(), err.data(), valid.data(), board_out.data(), &n_opt);
      if (st != ICC_OK) { std::cerr << "board point optimisation failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
      std::cout << "Optimized " << n_opt << " board points (observed in more than 30 views) and all view poses.\n";
    }
    st = icc_filter_bad_poses(h, nv, p.data(), valid.data());                  // app :66-67
    if (st != ICC_OK) { std::cerr << "pose filter failed (" << st << ")" << std::endl; return 2; }
    icc_destroy(h);
    Value out = Value::object(); out["views"] = Value::object(); out["tracks"] = Value::object();
    int kept = 0; double total = 0.0;
    for (int i = 0; i < nv; ++i) {
      if (!valid[i]) { std::cout << "Pose estimation failed or view rejected at timestamp " << sv.timestamp_us[i] * 1e-6 << "s from " << (sv.off[i + 1] - sv.off[i]) << " points.\n"; continue; }
      Value v = Value::object();
      v["q_wc"] = Value::array(); v["q_wc"].push_back(Value(q[4 * i + 3])); for (int d = 0; d < 3; ++d) v["q_wc"].push_back(Value(q[4 * i + d]));
      v["p_wc"] = Value::array(); for (int d = 0; d < 3; ++d) v["p_wc"].push_back(Value(p[3 * i + d]));
      v["timestamp_s"] = Value(sv.timestamp_us[i] * 1e-6); v["mean_reproj_error"] = Value(err[i]);
      out["views"][icccli::pose_view_name(sv.timestamp_us[i])] = v;
      ++kept; total += err[i];
    }
    for (int i = 0; i < np; ++i) { Value t = Value::array(); for (int d = 0; d < 4; ++d) t.push_back(Value(board_out[4 * i + d])); out["tracks"][std::to_string(i)] = t; }
    std::cout << "Estimated " << kept << " of " << nv << " view poses, mean " << (pose_error == ICC_POSE_ERROR_TANGENT ? "tangent" : "normalised") << " reprojection error " << (kept ? total / kept : 0.0) << "\n";
    if (!F.str["output_pose_dataset"].empty()) {
      std::ofstream f(F.str["output_pose_dataset"]);
      if (!f.is_open()) { std::cerr << "could not write " << F.str["output_pose_dataset"] << std::endl; return 1; }
      f << iccjson::dump(out, 1) << std::endl;
    }
  } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  return 0;
}
