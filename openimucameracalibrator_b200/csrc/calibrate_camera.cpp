// Drop-in host program for applications/calibrate_camera.cc of urbste/OpenImuCameraCalibrator (SURVEY.md §8(f) row f4): same
// gflags names and defaults (app :25-45), same input (UBJSON corner file of extract_board_to_json), same outputs:
//   <save_path_calib_dataset>.json          camera calibration in the layout of io::write_camera_calibration
//                                           (src/io/write_camera_calibration.cc:33-133) -- what every other tool reads back
//   <save_path_calib_dataset>.calibdata     the calibration dataset (views + board points)
// The calibration itself -- CameraCalibrator::CalibrateCameraFromJson / RunCalibration (src/core/camera_calibrator.cc:131-389) --
// runs on the GPU through icc_calibrate_camera; PrintResult (:391-458) is reproduced on stdout.
//
// Deliberate differences: the .calibdata file is the JSON pose dataset this repository's tools exchange ({"views": {"<name>":
// {"q_wc": [w,x,y,z], "p_wc": [...], "timestamp_s": t, "mean_reproj_error": e}}, "tracks": {...}}), not Theia's cereal binary
// (unreadable without Theia); the *_ransac_poses.ply / *_final_poses.ply point clouds are not written.  --optimize_board_points
// (camera_calibrator.cc:207-216) refines the board points on the GPU and writes them as the dataset's tracks.
// Extra flags: --device (CUDA ordinal, default 0); --pose_shutter global|rolling (default global): rolling calibrates with corners exposed row
// by row, line delay 1 / camera_fps / image_height of the corner file and the view velocities from the rolling-shutter pose step
// (icc_set_camcal_rolling_shutter, automatic mode).  The output files keep their layout.
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"

#include <cmath>
#include <fstream>
#include <iostream>

using iccjson::Value;

int main(int argc, char** argv) {
  icccli::Flags F;
  F.str = {{"input_corners", ""}, {"camera_model_to_calibrate", "DOUBLE_SPHERE"}, {"save_path_calib_dataset", ""}, {"pose_shutter", "global"}};
  F.boolean = {{"optimize_board_points", false}, {"verbose", false}};
  F.num = {{"grid_size", 0.04}, {"device", 0.0}};
  bool rolling = false;
  try { icccli::parse_flags(argc, argv, F); rolling = icccli::parse_pose_shutter(F.str["pose_shutter"]); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  try {
    Value scene_json; icccli::SceneViews sv;
    try { scene_json = icccli::load_scene(F.str["input_corners"], sv); } catch (const std::exception& e) { std::cerr << "Check failed: Failed to load " << F.str["input_corners"] << ": " << e.what() << std::endl; return 1; }
    const std::string model_name = F.str["camera_model_to_calibrate"];
    const icccli::CameraLayout* cam = icccli::find_camera(model_name);
    if (!cam) { std::cerr << "ERROR: unknown camera model '" << model_name << "'" << std::endl; return 1; }
    const int model = cam->id;
    const int width = (int)scene_json.at("image_width").num(), height = (int)scene_json.at("image_height").num();
    const double fps = scene_json.at("camera_fps").num();
    int np = 0;
    const std::vector<double> board = icccli::read_scene_points(scene_json, np);
    const int nv = (int)sv.timestamp_us.size();
    if (nv == 0) { std::cerr << "Check failed: the corner file holds no views" << std::endl; return 1; }
    double line_delay = 0.0;
    if (rolling) { try { line_delay = icccli::pose_line_delay(fps, height); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; } }
    icc_handle* h = nullptr;
    icc_status st = icc_create(&h, (int)F.num["device"]);
    if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    std::vector<double> q(4 * (size_t)nv), p(3 * (size_t)nv), err(nv), intr(ICC_MAX_INTRINSICS, 0.0); std::vector<int32_t> used(nv);
    icc_camcal_options opt{}; opt.grid_size = F.num["grid_size"]; opt.optimize_board_points = F.boolean["optimize_board_points"] ? 1 : 0;
    icc_camcal_summary S{};
    st = icc_set_board_points(h, np, board.data());
    std::vector<double> frame_t(nv);
    for (int i = 0; i < nv; ++i) frame_t[i] = sv.timestamp_us[i] * 1e-6;
    if (st == ICC_OK && rolling) st = icc_set_camcal_rolling_shutter(h, line_delay, nv, frame_t.data(), nullptr);
    if (st == ICC_OK) st = icc_calibrate_camera(h, model, width, height, nv, sv.off.data(), sv.ids.data(), sv.uv.data(), nullptr, nullptr, nullptr, 0.0, 0.0, &opt,
                                                intr.data(), q.data(), p.data(), err.data(), used.data(), &S);
    if (st != ICC_OK) { std::cerr << "camera calibration failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    std::vector<double> board_out(board);
    if (opt.optimize_board_points) icc_get_board_points(h, board_out.data(), np);
    if (rolling) {
      std::vector<double> vel(6 * (size_t)nv); int32_t n_static = 0;
      if (icc_get_camcal_velocities(h, nv, vel.data(), &n_static) == ICC_OK)
        std::cout << "Rolling shutter: line delay " << line_delay << " s, " << n_static << " valid views without a neighbour in time keep the global-shutter model.\n";
    }
    icc_destroy(h);
    std::cout << "Using " << S.n_views_selected << " views for camera calibration.\n";
    if (F.boolean["verbose"]) for (int i = 0; i < nv; ++i) if (used[i]) std::cout << "View: " << icccli::pose_view_name(sv.timestamp_us[i]) << " RMSE reprojection error: " << err[i] << "\n";
    if (opt.optimize_board_points && S.success) std::cout << "Optimized " << S.n_points_optimized << " board points.\n";
    if (!S.success) { std::cerr << "Not enough views for proper calibration!\nCalibration failed.\n"; return 3; }
    std::cout << "Final camera calibration reprojection error: " << S.final_reproj_error << " from " << S.n_views_used << " view." << std::endl;
    const std::string out = F.str["save_path_calib_dataset"];
    if (!out.empty()) {
      // io::write_camera_calibration (src/io/write_camera_calibration.cc:33-133)
      Value j = Value::object();
      j["stabelized"] = Value(false); j["fps"] = Value(fps); j["nr_calib_images"] = Value((int64_t)S.n_views_used); j["final_reproj_error"] = Value(S.final_reproj_error);
      j["image_width"] = Value((int64_t)width); j["image_height"] = Value((int64_t)height);   // integers, like io::write_camera_calibration
      j["intrinsic_type"] = Value(model_name);
      j["intrinsics"] = icccli::write_intrinsics(*cam, intr.data());
      std::ofstream f(out + ".json");
      if (!f.is_open()) { std::cerr << "Could not open: " << out << ".json\nCheck failed: Could not write calibration file.\n"; return 1; }
      f << iccjson::dump(j, 2) << std::endl;
      Value ds = Value::object(); ds["views"] = Value::object(); ds["tracks"] = Value::object();
      for (int i = 0; i < nv; ++i) {
        if (!used[i]) continue;
        Value v = Value::object();
        v["q_wc"] = Value::array(); v["q_wc"].push_back(Value(q[4 * i + 3])); for (int d = 0; d < 3; ++d) v["q_wc"].push_back(Value(q[4 * i + d]));
        v["p_wc"] = Value::array(); for (int d = 0; d < 3; ++d) v["p_wc"].push_back(Value(p[3 * i + d]));
        v["timestamp_s"] = Value(sv.timestamp_us[i] * 1e-6); v["mean_reproj_error"] = Value(err[i]);
        ds["views"][icccli::pose_view_name(sv.timestamp_us[i])] = v;
      }
      for (int i = 0; i < np; ++i) { Value t = Value::array(); for (int d = 0; d < 4; ++d) t.push_back(Value(board_out[4 * i + d])); ds["tracks"][std::to_string(i)] = t; }
      std::ofstream g(out + ".calibdata");
      if (!g.is_open()) { std::cerr << "could not write " << out << ".calibdata" << std::endl; return 1; }
      g << iccjson::dump(ds, 1) << std::endl;
      // theia::WritePlyFile(output_path + "_final_poses.ply", recon, camera colour (255, 0, 0), min 1 observation) (camera_calibrator.cc:381-384):
      // the camera positions of the views that took part, then the board points.  (The reference also dumps "_ransac_poses.ply" before the
      // calibration, :342-345; there is no RANSAC stage here -- the initial poses never leave the device.)
      std::ofstream ply(out + "_final_poses.ply");
      if (!ply.is_open()) { std::cerr << "could not write " << out << "_final_poses.ply" << std::endl; return 1; }
      int n_cam = 0; for (int i = 0; i < nv; ++i) n_cam += used[i] ? 1 : 0;
      ply << "ply\nformat ascii 1.0\nelement vertex " << n_cam + np << "\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n";
      for (int i = 0; i < nv; ++i) if (used[i]) ply << p[3 * i] << " " << p[3 * i + 1] << " " << p[3 * i + 2] << " 255 0 0\n";
      for (int i = 0; i < np; ++i) { const double w = board_out[4 * i + 3]; ply << board_out[4 * i] / w << " " << board_out[4 * i + 1] / w << " " << board_out[4 * i + 2] / w << " 255 255 255\n"; }
    }
    // CameraCalibrator::PrintResult (:391-458)
    icccli::print_camera(std::cout, *cam, intr.data());
  } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  return 0;
}
