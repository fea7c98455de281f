// Drop-in host program for applications/continuous_time_imu_to_camera_calibration.cc of urbste/OpenImuCameraCalibrator:
// same gflags names (app :38-80), same input files (UBJSON corners, camera / telemetry / init / bias / IMU-intrinsics /
// spline-weighting JSON), same result JSON keys (app :247-332) and the two PLY files (app :335-364); everything between
// "files parsed" and "results written" runs on the GPU through the C-ABI of include/icc_b200.h.
//
// One deliberate difference: --input_pose_dataset.  The reference reads Theia's cereal-binary .calibdata
// (theia::ReadReconstruction, app :95-97), which cannot be parsed without Theia.  This program reads the same content as
// JSON:  {"views": {"<view name>": {"q_wc": [w,x,y,z], "p_wc": [x,y,z]}}, "tracks": {"<id>": [x,y,z,w]}}
// where q_wc = R_cw^T and p_wc = camera position (what app :137-145 / impl.h:290-300 take from each theia::Camera).
// When --input_pose_dataset is omitted, the per-view board poses are estimated in-process on the GPU from the corner file
// (icc_estimate_board_poses = PoseEstimator::EstimatePosesFromJson, SURVEY.md §8(f) row f1), i.e. the corner file alone suffices;
// --pose_error normalized|tangent (default normalized) selects that step's residual (icc_set_pose_error: tangent keeps the corners of
// fisheye lenses beyond 90 degrees); --pose_shutter global|rolling (default global) its shutter (icc_set_pose_rolling_shutter: rolling gives each
// view's pose at its frame timestamp from row-timed corners, line delay 1 / fps / height).  --pose_shutter rolling with --global_shutter or
// with --input_pose_dataset is a usage error: the first contradicts it, the second skips the pose step.
// --reprojection_error pixel|tangent (default pixel) selects the vision residual of the spline solve (icc_set_reprojection_error: tangent
// scores every corner as its unit bearing, so that corners of wide lenses keep pulling wherever the camera model's projection would fail;
// the reported reprojection errors stay in pixels).  The rank processes of --gpus N re-execute this command line and so get the same residual.
// Extra flags (not in the reference): --device (CUDA ordinal, default 0), --parse_only (stop after parsing, print a summary),
// --gpus N (residual blocks sharded by time slice over devices device..device+N-1 of this host: the binary spawns one rank process per
// extra device -- hidden flags --shard_rank / --shard_world / --comm_id_hex -- each with the library's own NCCL communicator; one
// all-reduce of the packed normal equations per Jacobian evaluation).
// --outlier_sigma k (default 0 = off), --outlier_min_px m (default 1), --outlier_rounds n (default 2): after stage 1, up to n rounds of
// icc_reject_outlier_corners (corners whose reprojection error exceeds max(m, k * rms) leave the solve) each followed by stage 1 again with
// the same flags and iteration limit, until a round rejects nothing; stage 2 then runs as before.  With k > 0 the result JSON also holds
// "outlier_corners_rejected" (all rounds) and "outlier_threshold_px" (the last round's threshold).
// --bias_knot_spacing_s dt (default 10, the reference's), --accl_random_walk / --gyro_random_walk q (Kalibr's names and units, m/s^3/sqrt(Hz)
// and rad/s^2/sqrt(Hz), default 0 = no prior) or --imu_noise_json (the --output_json document of fit_allan_variance, per axis q = sqrt(3) |K| /
// scale): both bias splines at spacing dt with a random-walk prior of density q (icc_set_bias_splines, icc_set_bias_random_walk).  They act
// through --reestimate_biases only, so without it they are refused, as are the scalars together with the JSON.  When given, the tool prints
// the knot counts, spacing and densities, and the result JSON gains "bias_knot_spacing_s", "accl_random_walk" and "gyro_random_walk".
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"

#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <iostream>
#include <map>
#include <set>
#include <thread>
#include <spawn.h>
#include <sys/wait.h>
#include <unistd.h>

using iccjson::Value;

namespace {

icccli::Flags default_flags() {
  icccli::Flags f;
  f.str = {{"telemetry_json", ""}, {"input_pose_dataset", ""}, {"input_corners", ""}, {"camera_calibration_json", ""},
    {"gyro_to_cam_initial_calibration", ""}, {"imu_intrinsics", ""}, {"imu_bias_file", ""}, {"spline_error_weighting_json", ""}, {"output_path", ""},
    {"result_output_json", ""}, {"known_grav_dir_axis", "Z"}, {"debug_video_path", ""}, {"comm_id_hex", ""}, {"pose_error", "normalized"},
    {"pose_shutter", "global"}, {"reprojection_error", "pixel"}, {"imu_noise_json", ""}};
  f.boolean = {{"global_shutter", false}, {"calibrate_cam_line_delay", false}, {"reestimate_biases", false}, {"parse_only", false}, {"json_selftest", false}};
  f.num = {{"max_t", 1000.0}, {"gravity_const", 9.81}, {"device", 0.0}, {"gpus", 1.0}, {"shard_rank", 0.0}, {"shard_world", 1.0},
    {"outlier_sigma", 0.0}, {"outlier_min_px", 1.0}, {"outlier_rounds", 2.0}, {"bias_knot_spacing_s", 10.0}, {"accl_random_walk", 0.0}, {"gyro_random_walk", 0.0}};
  return f;
}

#define CHECK_MSG(cond, msg) do { if (!(cond)) { std::cerr << "Check failed: " #cond " " << msg << std::endl; std::exit(1); } } while (0)
#define ICC(call) do { icc_status s__ = (call); if (s__ != ICC_OK) { std::cerr << #call << " failed (" << s__ << "): " << icc_last_error(h) << std::endl; std::exit(2); } } while (0)

int grav_dir_string_to_int(const std::string& s) {   // src/utils/utils.cc:150-161
  if (s == "UNKNOWN") return -1;
  if (s == "X") return 0;
  if (s == "Y") return 1;
  if (s == "Z") return 2;
  return -1;
}

void write_ply(const std::string& path, const std::vector<std::array<double, 3>>& pts, const std::vector<std::array<int, 3>>& col) {
  std::ofstream f(path);
  if (!f.is_open()) throw std::runtime_error("could not write " + path);
  f << "ply\nformat ascii 1.0\nelement vertex " << pts.size() << "\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n";
  for (size_t i = 0; i < pts.size(); ++i) f << pts[i][0] << " " << pts[i][1] << " " << pts[i][2] << " " << col[i][0] << " " << col[i][1] << " " << col[i][2] << "\n";
}

Value xyz(double x, double y, double z) { Value v = Value::object(); v["x"] = Value(x); v["y"] = Value(y); v["z"] = Value(z); return v; }

}  // namespace

// Result JSON (app :247-332) streamed through iccjson::Writer: `head` holds every key but the trajectory (all of them sort before it),
// the trajectory object -- 100 k entries of six xyz objects for a 100 s sequence, ~90 MB of text -- is emitted straight from the arrays
// in std::map<std::string> key order (lexicographic on the decimal timestamp; a repeated timestamp keeps the last sample), i.e. the bytes
// nlohmann::json / the tree route would produce, without building 700 k tree nodes.
static void write_result(iccjson::Writer& w, const Value& head, int n_used, const int64_t* t_ns, const double* ug, const double* gs, const double* gb,
                         const double* ua, const double* as, const double* ab, int threads = 0) {
  w.begin_object();
  for (const auto& kv : *head.o) { w.key(kv.first); w.value(kv.second); }
  if (n_used) {
    const bool tr = getenv("ICC_JSON_TRACE") != nullptr; auto T0 = std::chrono::steady_clock::now();   // ICC_JSON_TRACE=1: phase times to stderr
    auto lap = [&](const char* what) { if (tr) { auto T1 = std::chrono::steady_clock::now(); std::cerr << "    [json] " << what << " " << std::chrono::duration<double, std::milli>(T1 - T0).count() << " ms\n"; T0 = T1; } };
    std::vector<std::pair<std::string, int>> keys(n_used);
    for (int i = 0; i < n_used; ++i) keys[i] = {std::to_string(t_ns[i]), i};
    std::stable_sort(keys.begin(), keys.end(), [](const std::pair<std::string, int>& a, const std::pair<std::string, int>& b) { return a.first < b.first; });
    lap("keys + sort");
    w.key("trajectory"); w.begin_object();
    // The entries are formatted by several threads, each into its own fragment that continues inside the two open objects (root, trajectory);
    // the fragments are then written in order.  ~900 bytes of text per entry: formatting, not the file system, is the cost of this file.
    auto emitted = [&](int k) { return !(k + 1 < n_used && keys[k + 1].first == keys[k].first); };   // a repeated timestamp keeps the last sample
    if (threads <= 0) threads = (int)std::min<unsigned>(8, std::max<unsigned>(1, std::thread::hardware_concurrency()));
    threads = std::max(1, std::min(threads, n_used / 64 + 1));
    std::vector<int> cut(threads + 1), before(threads + 1, 0);
    for (int c = 0; c <= threads; ++c) cut[c] = (int)((int64_t)n_used * c / threads);
    for (int c = 0; c < threads; ++c) { int e = 0; for (int k = cut[c]; k < cut[c + 1]; ++k) e += emitted(k); before[c + 1] = before[c] + e; }
    std::vector<std::string> frag(threads);
    auto work = [&](int c) {
      std::string& out = frag[c]; out.reserve((size_t)(before[c + 1] - before[c]) * 960 + 64);
      iccjson::Writer fw(4, &out, std::vector<size_t>{1, (size_t)before[c]});
      auto xyz_at = [&](const char* k, const double* v, int i) { fw.key(k); fw.begin_object(); fw.key("x"); fw.value(v[3 * i]); fw.key("y"); fw.value(v[3 * i + 1]); fw.key("z"); fw.value(v[3 * i + 2]); fw.end_object(); };
      for (int k = cut[c]; k < cut[c + 1]; ++k) {
        if (!emitted(k)) continue;
        const int i = keys[k].second;
        fw.key(keys[k].first); fw.begin_object();
        xyz_at("accl_bias", ab, i); xyz_at("accl_imu", ua, i); xyz_at("accl_spline", as, i); xyz_at("gyro_bias", gb, i); xyz_at("gyro_imu", ug, i); xyz_at("gyro_spline", gs, i);
        fw.end_object();
      }
    };
    std::vector<std::thread> pool;
    for (int c = 1; c < threads; ++c) pool.emplace_back(work, c);
    work(0);
    for (auto& t : pool) t.join();
    lap("format");
    for (int c = 0; c < threads; ++c) w.raw_members(frag[c], (size_t)(before[c + 1] - before[c]));
    lap("concatenate / write");
    w.end_object();
  }
  w.end_object();
}

// --json_selftest: the streamed result equals the tree route byte for byte (random samples incl. repeated and unordered timestamps)
static int json_selftest() {
  const int n = 257;
  std::vector<int64_t> t(n); std::vector<double> a[6]; for (auto& v : a) v.resize(3 * n);
  uint64_t s = 88172645463325252ull; auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  for (int i = 0; i < n; ++i) { t[i] = (int64_t)(rnd() % 5000) * 1000003; for (auto& v : a) for (int d = 0; d < 3; ++d) v[3 * i + d] = (double)(int64_t)(rnd() % 2000001 - 1000000) * (i % 7 == 0 ? 1.0 : 1e-6); }
  t[5] = t[4]; t[100] = 7;
  Value head = Value::object(); head["final_reproj_error"] = Value(0.25); head["q_i_c"] = xyz(1, 2, 3); head["time_offset_imu_to_cam_s"] = Value(-0.0123);
  Value tree = head, traj = Value::object();
  tree = Value::object(); for (const auto& kv : *head.o) tree[kv.first] = kv.second;
  for (int i = 0; i < n; ++i) {
    Value e = Value::object();
    e["gyro_imu"] = xyz(a[0][3 * i], a[0][3 * i + 1], a[0][3 * i + 2]); e["gyro_spline"] = xyz(a[1][3 * i], a[1][3 * i + 1], a[1][3 * i + 2]); e["gyro_bias"] = xyz(a[2][3 * i], a[2][3 * i + 1], a[2][3 * i + 2]);
    e["accl_imu"] = xyz(a[3][3 * i], a[3][3 * i + 1], a[3][3 * i + 2]); e["accl_spline"] = xyz(a[4][3 * i], a[4][3 * i + 1], a[4][3 * i + 2]); e["accl_bias"] = xyz(a[5][3 * i], a[5][3 * i + 1], a[5][3 * i + 2]);
    traj[std::to_string(t[i])] = e;
  }
  tree["trajectory"] = traj;
  std::string streamed;
  bool same = true;
  const std::string want = iccjson::dump(tree, 4);
  for (int threads : {1, 2, 3, 5, 8}) {   // the fragments of any number of formatting threads concatenate to the tree route's bytes
    streamed.clear();
    { iccjson::Writer w(4, &streamed); write_result(w, head, n, t.data(), a[0].data(), a[1].data(), a[2].data(), a[3].data(), a[4].data(), a[5].data(), threads); }
    same = same && streamed == want;
  }
  std::cout << (same ? "json selftest ok: " : "json selftest FAILED: ") << streamed.size() << " bytes" << std::endl;
  if (const char* big = getenv("ICC_JSON_SELFTEST_N")) {   // formatting time of a config-4-sized trajectory (100 k entries) per thread count
    const int m = atoi(big);
    std::vector<int64_t> tb(m); std::vector<double> ab[6]; for (auto& v : ab) v.resize(3 * (size_t)m);
    for (int i = 0; i < m; ++i) { tb[i] = 1000000 * (int64_t)i + 123; for (auto& v : ab) for (int d = 0; d < 3; ++d) v[3 * (size_t)i + d] = (double)(int64_t)(rnd() % 2000001 - 1000000) * 1.0000001e-6; }
    for (int threads : {1, 2, 4, 8}) {
      std::string out; const auto t0 = std::chrono::steady_clock::now();
      { iccjson::Writer w(4, &out); write_result(w, head, m, tb.data(), ab[0].data(), ab[1].data(), ab[2].data(), ab[3].data(), ab[4].data(), ab[5].data(), threads); }
      std::cout << "  " << m << " entries, " << threads << " formatting thread(s): " << std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() << " ms, " << out.size() << " bytes" << std::endl;
    }
  }
  return same ? 0 : 1;
}

int main(int argc, char** argv) {
  icccli::Flags F = default_flags();
  int pose_error = ICC_POSE_ERROR_NORMALIZED, reproj_error = ICC_REPROJ_ERROR_PIXEL;
  bool pose_rolling = false;
  double outlier_sigma = 0.0, outlier_min_px = 1.0; int outlier_rounds = 2;
  bool bias_walk = false; double bias_dt = 10.0, acc_q[3] = {0, 0, 0}, gyr_q[3] = {0, 0, 0};   // --bias_knot_spacing_s / --*_random_walk / --imu_noise_json
  try {
    icccli::parse_flags(argc, argv, F); pose_error = icccli::parse_pose_error(F.str["pose_error"]); pose_rolling = icccli::parse_pose_shutter(F.str["pose_shutter"]);
    reproj_error = icccli::parse_reprojection_error(F.str["reprojection_error"]);
    outlier_sigma = F.num["outlier_sigma"]; outlier_min_px = F.num["outlier_min_px"];
    if (!(outlier_sigma >= 0.0) || !std::isfinite(outlier_sigma)) throw std::runtime_error("--outlier_sigma must be a finite number >= 0 (0 = off)");
    if (!(outlier_min_px >= 0.0) || !std::isfinite(outlier_min_px)) throw std::runtime_error("--outlier_min_px must be a finite number >= 0");
    if (!(F.num["outlier_rounds"] >= 0.0) || F.num["outlier_rounds"] > 1000.0 || F.num["outlier_rounds"] != std::floor(F.num["outlier_rounds"]))
      throw std::runtime_error("--outlier_rounds must be a whole number >= 0");
    outlier_rounds = (int)F.num["outlier_rounds"];
    bias_dt = F.num["bias_knot_spacing_s"];
    const double aq = F.num["accl_random_walk"], gq = F.num["gyro_random_walk"];
    if (!(bias_dt > 0.0) || !std::isfinite(bias_dt)) throw std::runtime_error("--bias_knot_spacing_s must be a finite number > 0");
    if (!(aq >= 0.0) || !std::isfinite(aq) || !(gq >= 0.0) || !std::isfinite(gq)) throw std::runtime_error("--accl_random_walk / --gyro_random_walk must be finite numbers >= 0 (0 = no prior)");
    const bool scalars = aq > 0.0 || gq > 0.0, noise_json = !F.str["imu_noise_json"].empty();
    if (scalars && noise_json) throw std::runtime_error("--imu_noise_json and --accl_random_walk / --gyro_random_walk both give the random-walk densities: use one");
    bias_walk = scalars || noise_json || bias_dt != 10.0;
    if (bias_walk && !F.boolean["reestimate_biases"])
      throw std::runtime_error("--bias_knot_spacing_s, --accl_random_walk, --gyro_random_walk and --imu_noise_json shape the bias splines, which only --reestimate_biases frees: add it");
    for (int a = 0; a < 3; ++a) { acc_q[a] = aq; gyr_q[a] = gq; }
    if (noise_json) icccli::bias_random_walk_from_allan(iccjson::load_json(F.str["imu_noise_json"]), acc_q, gyr_q);
    if (pose_rolling && F.boolean["global_shutter"]) throw std::runtime_error("--pose_shutter rolling contradicts --global_shutter");
    if (pose_rolling && !F.str["input_pose_dataset"].empty()) throw std::runtime_error("--pose_shutter rolling applies to the in-process pose step, which --input_pose_dataset skips");
  } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  const double S_TO_NS = 1e9, US_TO_S = 1e-6, S_TO_US = 1e6, NS_TO_S = 1e-9;
  if (F.boolean["json_selftest"]) return json_selftest();
  try {
    // ---- inputs (app :93-184) ---------------------------------------------------------------------------------------
    const bool have_poses = !F.str["input_pose_dataset"].empty();
    Value pose_dataset;
    if (have_poses) {
      try { pose_dataset = iccjson::load_json(F.str["input_pose_dataset"]); }
      catch (const std::exception& e) { CHECK_MSG(false, "Could not read Reconstruction file (JSON pose dataset expected, Theia .calibdata is not supported): " << e.what()); }
    }
    Value scene_json; icccli::SceneViews sv;
    try { scene_json = icccli::load_scene(F.str["input_corners"], sv); } catch (const std::exception& e) { CHECK_MSG(false, "Failed to load " << F.str["input_corners"] << ": " << e.what()); }
    std::vector<double> intr; int width = 0, height = 0; double fps = 0;
    int model = -1;
    try { model = icccli::read_camera(iccjson::load_json(F.str["camera_calibration_json"]), intr, width, height, fps); }
    catch (const std::exception& e) { CHECK_MSG(false, "Could not read camera calibration: " << F.str["camera_calibration_json"] << ": " << e.what()); }
    // board tracks come from the pose dataset (possibly refined), app :108-119; without one, from the corner file's scene_pts
    int max_id = -1;
    std::vector<double> board;
    if (have_poses) {
      const Value& tracks = pose_dataset.at("tracks");
      for (const auto& kv : *tracks.o) max_id = std::max(max_id, std::stoi(kv.first));
      board.assign(4 * (size_t)(max_id + 1), 0.0);
      for (int i = 0; i <= max_id; ++i) board[4 * i + 3] = 1.0;
      for (const auto& kv : *tracks.o) { const int id = std::stoi(kv.first); for (int d = 0; d < 4; ++d) board[4 * id + d] = kv.second.at(d).num(); }
    } else {
      int np = 0; board = icccli::read_scene_points(scene_json, np); max_id = np - 1;
    }
    // telemetry (src/io/read_telemetry.cc:29-69)
    icccli::Telemetry tel;
    try { tel = icccli::load_telemetry(F.str["telemetry_json"]); } catch (const std::exception& e) { CHECK_MSG(false, "Could not read: " << F.str["telemetry_json"] << ": " << e.what()); }
    CHECK_MSG(tel.gyr.size() == 3 * tel.t_ns.size() && tel.acc.size() == 3 * tel.t_ns.size(), "Telemetry should have the same amount of timestamps, accelerometer and gyroscope values.");
    std::vector<double> imu_t(tel.t_ns.size());
    for (size_t i = 0; i < imu_t.size(); ++i) imu_t[i] = tel.t_ns[i] * NS_TO_S;
    const std::vector<double>& acc = tel.acc; const std::vector<double>& gyr = tel.gyr;
    double t_offset_cam_s = 0.0;
    if (!tel.img_t_ns.empty()) t_offset_cam_s = tel.img_t_ns[0] * NS_TO_S;
    // views: join corners with poses by name = to_string((uint64) timestamp_us)   (app :131-161)
    std::vector<double> frame_t, uv, q_wc, p_wc; std::vector<int32_t> off{0}, ids;
    int n_view_fallback = 0, n_view_dropped = 0;
    if (have_poses) {
      const Value& pviews = pose_dataset.at("views");
      for (size_t vi = 0; vi < sv.key.size(); ++vi) {
        const double timestamp_us = sv.timestamp_us[vi];
        // the pose tools name a view to_string((uint64)(ts * 1e-6 * 1e6)): that round trip can land one microsecond below the key
        // used here (the reference has the same mismatch and silently drops such views): fall back to the neighbouring names
        std::string view_name = std::to_string((uint64_t)timestamp_us);
        if (!pviews.contains(view_name)) {
          const std::string lo = std::to_string((uint64_t)timestamp_us - 1), hi = std::to_string((uint64_t)timestamp_us + 1);
          if (pviews.contains(lo)) { view_name = lo; ++n_view_fallback; } else if (pviews.contains(hi)) { view_name = hi; ++n_view_fallback; } else { ++n_view_dropped; continue; }
        }
        const Value& pv = pviews.at(view_name);
        frame_t.push_back(timestamp_us * US_TO_S + t_offset_cam_s);
        const Value& q = pv.at("q_wc");   // [w, x, y, z]
        q_wc.push_back(q.at(1).num()); q_wc.push_back(q.at(2).num()); q_wc.push_back(q.at(3).num()); q_wc.push_back(q.at(0).num());
        for (int d = 0; d < 3; ++d) p_wc.push_back(pv.at("p_wc").at(d).num());
        for (int cidx = sv.off[vi]; cidx < sv.off[vi + 1]; ++cidx) { ids.push_back(sv.ids[cidx]); uv.push_back(sv.uv[2 * cidx]); uv.push_back(sv.uv[2 * cidx + 1]); }
        off.push_back((int32_t)ids.size());
      }
    } else if (!F.boolean["parse_only"]) {
      // no pose dataset: estimate the per-view poses on the GPU and keep the views the reference's PoseEstimator would keep
      const int nv = (int)sv.timestamp_us.size();
      CHECK_MSG(nv > 0, "the corner file holds no views");
      icc_handle* hp = nullptr;
      { icc_status st = icc_create(&hp, (int)F.num["device"]); if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(hp) << std::endl; return 2; } }
      std::vector<double> q_all(4 * (size_t)nv), p_all(3 * (size_t)nv), err(nv); std::vector<int32_t> valid(nv);
      icc_status st = icc_set_camera(hp, model, intr.data(), (int)intr.size(), width, height);
      if (st == ICC_OK) st = icc_set_board_points(hp, max_id + 1, board.data());
      if (st == ICC_OK) st = icc_set_pose_error(hp, pose_error);
      std::vector<double> view_t(nv);
      for (int i = 0; i < nv; ++i) view_t[i] = sv.timestamp_us[i] * US_TO_S + t_offset_cam_s;
      if (st == ICC_OK && pose_rolling) {
        double ld = 0.0;
        try { ld = icccli::pose_line_delay(fps, height); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
        st = icc_set_pose_rolling_shutter(hp, ld, nv, view_t.data());
      }
      if (st == ICC_OK) st = icc_estimate_board_poses(hp, nv, sv.off.data(), sv.ids.data(), sv.uv.data(), 0.0, 0, q_all.data(), p_all.data(), err.data(), valid.data());
      if (st == ICC_OK) st = icc_filter_bad_poses(hp, nv, p_all.data(), valid.data());   // the pose app's last step (PoseEstimator::FilterBadPoses)
      if (st != ICC_OK) { std::cerr << "board pose estimation failed (" << st << "): " << icc_last_error(hp) << std::endl; return 2; }
      if (pose_rolling) {
        std::vector<double> vel(6 * (size_t)nv); int32_t n_static = 0;
        if (icc_get_pose_velocities(hp, nv, vel.data(), &n_static) == ICC_OK)
          std::cout << "Rolling-shutter board poses: " << n_static << " valid views without a neighbour in time keep the global-shutter model\n";
      }
      icc_destroy(hp);
      int kept = 0;
      for (int i = 0; i < nv; ++i) {
        if (!valid[i]) continue;
        ++kept;
        frame_t.push_back(sv.timestamp_us[i] * US_TO_S + t_offset_cam_s);
        for (int d = 0; d < 4; ++d) q_wc.push_back(q_all[4 * i + d]);
        for (int d = 0; d < 3; ++d) p_wc.push_back(p_all[3 * i + d]);
        for (int c = sv.off[i]; c < sv.off[i + 1]; ++c) { ids.push_back(sv.ids[c]); uv.push_back(sv.uv[2 * c]); uv.push_back(sv.uv[2 * c + 1]); }
        off.push_back((int32_t)ids.size());
      }
      std::cout << "Estimated board poses for " << kept << " of " << nv << " views on the GPU (no --input_pose_dataset given)\n";
    } else {
      for (size_t i = 0; i < sv.timestamp_us.size(); ++i) frame_t.push_back(sv.timestamp_us[i] * US_TO_S + t_offset_cam_s);
      ids = sv.ids; uv = sv.uv; off = sv.off;
    }
    CHECK_MSG(!frame_t.empty(), "no view of the corner file has a pose in the pose dataset");
    if (have_poses && !F.boolean["parse_only"]) {
      std::cout << "Views with a pose: " << frame_t.size() << " of " << sv.key.size() << " (" << n_view_fallback << " matched through a neighbouring microsecond name, " << n_view_dropped << " dropped)\n";
      if (n_view_dropped > 0) std::cerr << "WARNING: " << n_view_dropped << " views of the corner file have no pose in the pose dataset and are skipped\n";
    }
    // gyro-to-camera initialisation (src/io/read_misc.cc:63-82): T_i_c_init = (q_gyro_to_cam^-1, 0)   (app :164-170)
    Value init;
    try { init = iccjson::load_json(F.str["gyro_to_cam_initial_calibration"]); } catch (const std::exception& e) { CHECK_MSG(false, "Could not read: " << F.str["gyro_to_cam_initial_calibration"] << ": " << e.what()); }
    const Value& gq = init.at("gyro_to_camera_rotation");
    const double time_offset_imu_to_cam = init.at("time_offset_gyro_to_cam").num();
    icc_init_params ip; memset(&ip, 0, sizeof ip);
    ip.T_i_c_init[0] = -gq.at("x").num(); ip.T_i_c_init[1] = -gq.at("y").num(); ip.T_i_c_init[2] = -gq.at("z").num(); ip.T_i_c_init[3] = gq.at("w").num();
    // IMU intrinsics + biases (src/io/read_misc.cc:84-150)
    double acc_i[6] = {0, 0, 0, 1, 1, 1}, gyr_i[9] = {0, 0, 0, 0, 0, 0, 1, 1, 1};
    if (!F.str["imu_bias_file"].empty()) {
      try { Value b = iccjson::load_json(F.str["imu_bias_file"]); const char* ax[3] = {"x", "y", "z"}; for (int d = 0; d < 3; ++d) { ip.acc_bias[d] = b.at("accl_bias").at(ax[d]).num(); ip.gyr_bias[d] = b.at("gyro_bias").at(ax[d]).num(); } }
      catch (const std::exception& e) { std::cerr << "Error loading IMU bias file: " << F.str["imu_bias_file"] << " (" << e.what() << ")\n"; }
    }
    if (!F.str["imu_intrinsics"].empty()) {
      Value ii;
      try { ii = iccjson::load_json(F.str["imu_intrinsics"]); } catch (const std::exception& e) { CHECK_MSG(false, "Could not open " << F.str["imu_intrinsics"] << ": " << e.what()); }
      const Value& ma = ii.at("accelerometer").at("misalignment_matrix"); const Value& sa = ii.at("accelerometer").at("scale_matrix");
      // mis = [[1,-yz,zy],[xz,1,-zx],[-xy,yx,1]]  (utils/types.h:238-246)
      acc_i[0] = -ma.at(0).at(1).num(); acc_i[1] = ma.at(0).at(2).num(); acc_i[2] = -ma.at(1).at(2).num();
      acc_i[3] = sa.at(0).at(0).num(); acc_i[4] = sa.at(1).at(1).num(); acc_i[5] = sa.at(2).at(2).num();
      const Value& mg = ii.at("gyroscope").at("misalignment_matrix"); const Value& sg = ii.at("gyroscope").at("scale_matrix");
      gyr_i[0] = -mg.at(0).at(1).num(); gyr_i[1] = mg.at(0).at(2).num(); gyr_i[2] = -mg.at(1).at(2).num();
      gyr_i[3] = mg.at(1).at(0).num(); gyr_i[4] = -mg.at(2).at(0).num(); gyr_i[5] = mg.at(2).at(1).num();
      gyr_i[6] = sg.at(0).at(0).num(); gyr_i[7] = sg.at(1).at(1).num(); gyr_i[8] = sg.at(2).at(2).num();
    }
    memcpy(ip.acc_intrinsics, acc_i, sizeof acc_i); memcpy(ip.gyr_intrinsics, gyr_i, sizeof gyr_i);
    CHECK_MSG(!F.str["spline_error_weighting_json"].empty(), "You need to provide spline error weighting factors. Create with get_sew_for_dataset.py.");
    Value sew;
    try { sew = iccjson::load_json(F.str["spline_error_weighting_json"]); } catch (const std::exception& e) { CHECK_MSG(false, "Could not open " << F.str["spline_error_weighting_json"] << ": " << e.what()); }
    ip.dt_r3_s = sew.at("r3").at("knot_spacing").num(); ip.dt_so3_s = sew.at("so3").at("knot_spacing").num();
    ip.std_r3 = sew.at("r3").at("weighting_factor").num(); ip.std_so3 = sew.at("so3").at("weighting_factor").num();
    ip.time_offset_imu_to_cam_s = time_offset_imu_to_cam;
    double init_line_delay = 1. / fps / height;       // seconds despite the reference's "_us" name (app :186)
    if (F.boolean["global_shutter"]) init_line_delay = 0.0;
    ip.init_line_delay_s = init_line_delay;
    ip.dispatch_fov = model == ICC_CAM_FOV ? 1 : 0;

    if (F.boolean["parse_only"]) {
      Value s = Value::object();
      s["views"] = Value((int64_t)frame_t.size()); s["corners"] = Value((int64_t)ids.size()); s["imu_samples"] = Value((int64_t)imu_t.size());
      s["board_points"] = Value((int64_t)(max_id + 1)); s["camera_model"] = Value(model); s["intrinsics"] = Value::array();
      for (double v : intr) s["intrinsics"].push_back(Value(v));
      if (outlier_sigma > 0.0) { s["outlier_sigma"] = Value(outlier_sigma); s["outlier_min_px"] = Value(outlier_min_px); s["outlier_rounds"] = Value((int64_t)outlier_rounds); }
      if (bias_walk) {
        s["bias_knot_spacing_s"] = Value(bias_dt); s["accl_random_walk"] = Value::array(); s["gyro_random_walk"] = Value::array();
        for (int a = 0; a < 3; ++a) { s["accl_random_walk"].push_back(Value(acc_q[a])); s["gyro_random_walk"].push_back(Value(gyr_q[a])); }
      }
      s["init_line_delay_s"] = Value(init_line_delay); s["dt_so3"] = Value(ip.dt_so3_s); s["dt_r3"] = Value(ip.dt_r3_s); s["first_view_t_s"] = Value(frame_t.front());
      s["uv_sum"] = Value([&] { double a = 0; for (double v : uv) a += v; return a; }());
      // order-sensitive digests: the views must arrive in std::map key order, the corners of a view in the order of their id strings
      s["uv_order_digest"] = Value([&] { double a = 0; for (size_t i = 0; i < uv.size(); ++i) a += double(i % 1013 + 1) * uv[i]; return a; }());
      s["ids_order_digest"] = Value([&] { double a = 0; for (size_t i = 0; i < ids.size(); ++i) a += double(i % 1009 + 1) * ids[i]; return a; }());
      s["frame_t_digest"] = Value([&] { double a = 0; for (size_t i = 0; i < frame_t.size(); ++i) a += double(i % 101 + 1) * frame_t[i]; return a; }());
      s["imu_digest"] = Value([&] { double a = 0; for (size_t i = 0; i < imu_t.size(); ++i) a += double(i % 1013 + 1) * (imu_t[i] + acc[3 * i] + 2 * acc[3 * i + 1] + 3 * acc[3 * i + 2] + 5 * gyr[3 * i] + 7 * gyr[3 * i + 1] + 11 * gyr[3 * i + 2]); return a; }());
      std::cout << iccjson::dump(s) << std::endl;
      return 0;
    }

    // ---- solve on the GPU (app :188-221) ------------------------------------------------------------------------------
    icc_handle* h = nullptr;
    { icc_status s = icc_create(&h, (int)F.num["device"]); if (s != ICC_OK) { std::cerr << "icc_create failed (" << s << "): " << icc_last_error(h) << std::endl; return 2; } }
    ICC(icc_set_camera(h, model, intr.data(), (int)intr.size(), width, height));
    ICC(icc_set_reprojection_error(h, reproj_error));
    ICC(icc_set_board_points(h, max_id + 1, board.data()));
    ICC(icc_set_frames(h, (int)frame_t.size(), frame_t.data(), off.data(), ids.data(), uv.data(), q_wc.data(), p_wc.data()));
    ICC(icc_set_imu(h, (int)imu_t.size(), imu_t.data(), acc.data(), gyr.data()));
    if (bias_walk) {   // a sensor whose density is 0 keeps no prior
      ICC(icc_set_bias_splines(h, bias_dt, bias_dt));
      ICC(icc_set_bias_random_walk(h, acc_q[0] > 0.0 ? acc_q : nullptr, gyr_q[0] > 0.0 ? gyr_q : nullptr));
    }
    ICC(icc_batch_init_spline(h, &ip));
    if (bias_walk) {
      int nba = 0, nbg = 0; ICC(icc_get_num_knots(h, nullptr, nullptr, &nba, &nbg));
      std::cout << "Bias splines: " << nba << " accelerometer and " << nbg << " gyroscope knots at " << bias_dt << " s spacing; random walk accel ["
                << acc_q[0] << ", " << acc_q[1] << ", " << acc_q[2] << "] m/s^3/sqrt(Hz), gyro [" << gyr_q[0] << ", " << gyr_q[1] << ", " << gyr_q[2] << "] rad/s^2/sqrt(Hz)\n";
    }
    const int grav_dir_axis = grav_dir_string_to_int(F.str["known_grav_dir_axis"]);
    int flags = ICC_FLAG_SPLINE | ICC_FLAG_T_I_C;
    if (F.boolean["reestimate_biases"]) flags |= ICC_FLAG_IMU_BIASES;
    if (grav_dir_axis != -1) {
      double g[3] = {0, 0, 0}; g[grav_dir_axis] = F.num["gravity_const"];
      ICC(icc_set_known_gravity_dir(h, g));
      std::cout << "Setting a-priori gravity direction supplied by the user to: " << g[0] << " " << g[1] << " " << g[2] << "\n";
    } else flags |= ICC_FLAG_GRAVITY_DIR;
    // --gpus N: the binary re-executes itself once per extra device (rank r on device + r) with the NCCL id on the command line;
    // every rank parses the same files, keeps its own time slice of the residual blocks and runs the same optimisation calls (the
    // collectives are inside them).  Rank 0 (this process, or the one that was given --shard_rank 0) writes the results.
    const int n_gpus = std::max(1, (int)F.num["gpus"]);
    int shard_rank = (int)F.num["shard_rank"], shard_world = (int)F.num["shard_world"];
    if (shard_rank > 0) std::cout.setstate(std::ios::failbit);     // spawned ranks stay quiet
    const bool stage2 = F.boolean["calibrate_cam_line_delay"] && !F.boolean["global_shutter"];
    icc_comm* comm = nullptr;
    std::vector<pid_t> children;
    unsigned char comm_id[ICC_COMM_ID_BYTES];
    if (shard_world > 1) {                                  // spawned rank: the id arrives as hex
      const std::string hex = F.str["comm_id_hex"];
      CHECK_MSG(hex.size() == 2 * ICC_COMM_ID_BYTES, "--comm_id_hex must carry " << ICC_COMM_ID_BYTES << " bytes");
      for (int i = 0; i < ICC_COMM_ID_BYTES; ++i) comm_id[i] = (unsigned char)std::stoi(hex.substr(2 * (size_t)i, 2), nullptr, 16);
    } else if (n_gpus > 1) {                                // launcher = rank 0
      if (icc_comm_unique_id(comm_id) != ICC_OK) { std::cerr << "icc_comm_unique_id failed: " << icc_comm_last_error() << std::endl; return 2; }
      std::string hex; char b2[3];
      for (int i = 0; i < ICC_COMM_ID_BYTES; ++i) { snprintf(b2, sizeof b2, "%02x", comm_id[i]); hex += b2; }
      shard_rank = 0; shard_world = n_gpus;
      for (int r = 1; r < n_gpus; ++r) {
        std::vector<std::string> av(argv, argv + argc);
        av.push_back("--gpus=1"); av.push_back("--shard_rank=" + std::to_string(r)); av.push_back("--shard_world=" + std::to_string(n_gpus));
        av.push_back("--device=" + std::to_string((int)F.num["device"] + r)); av.push_back("--comm_id_hex=" + hex);
        std::vector<char*> cav; for (auto& a : av) cav.push_back(const_cast<char*>(a.c_str())); cav.push_back(nullptr);
        pid_t pid = 0;
        if (posix_spawn(&pid, "/proc/self/exe", nullptr, nullptr, cav.data(), environ) != 0) { std::cerr << "could not spawn rank " << r << std::endl; return 2; }
        children.push_back(pid);
      }
      std::cout << "Residual blocks sharded over " << n_gpus << " GPUs, one rank process each (NCCL " << icc_comm_nccl_version() << ")\n";
    }
    icc_summary s1, s2;
    if (shard_world > 1) {
      if (icc_comm_create(&comm, comm_id, shard_rank, shard_world, (int)F.num["device"]) != ICC_OK) { std::cerr << "icc_comm_create failed: " << icc_comm_last_error() << std::endl; return 2; }
      ICC(icc_set_comm(h, comm));
      ICC(icc_batch_init_spline(h, &ip));               // again, now with this rank's shard
      if (grav_dir_axis != -1) { double g[3] = {0, 0, 0}; g[grav_dir_axis] = F.num["gravity_const"]; ICC(icc_set_known_gravity_dir(h, g)); }
    }
    ICC(icc_optimize(h, 50, flags, &s1));
    // --outlier_sigma: reject, and solve stage 1 again, until a round rejects nothing (every rank runs the same calls: the threshold is global)
    int64_t outliers_rejected = 0; double outlier_threshold = 0.0;
    for (int round = 1; outlier_sigma > 0.0 && round <= outlier_rounds; ++round) {
      icc_outlier_summary os;
      ICC(icc_reject_outlier_corners(h, outlier_sigma, outlier_min_px, &os));
      outliers_rejected += os.n_rejected; outlier_threshold = os.threshold_px;
      std::cout << "Outlier round " << round << ": threshold " << os.threshold_px << " px, rejected " << os.n_rejected << " of " << os.n_corners
                << " corners (" << os.n_failed << " failed projections, " << os.n_frames_emptied << " views emptied)\n";
      if (os.n_rejected == 0) break;
      ICC(icc_optimize(h, 50, flags, &s1));
    }
    if (stage2) ICC(icc_optimize(h, 10, ICC_FLAG_CAM_LINE_DELAY, &s2));
    if (shard_rank > 0) { icc_destroy(h); icc_comm_destroy(comm); return 0; }   // only rank 0 reports
    double reproj_error = s1.mean_reproj_error, reproj_error_after_ld = stage2 ? s2.mean_reproj_error : reproj_error;
    std::cout << "LM iterations: " << s1.iterations << " cost " << s1.initial_cost << " -> " << s1.final_cost << "  (" << s1.seconds_total << " s, " << s1.gpu_launches << " kernel launches)\n";
    std::cout << "Mean reprojection error " << reproj_error << "px\nMean reprojection error after line delay optim " << reproj_error_after_ld << "px\n";

    // ---- results (app :226-332) ---------------------------------------------------------------------------------------
    double T[7], g[3], ld;
    ICC(icc_get_T_i_c(h, T)); ICC(icc_get_gravity(h, g)); ICC(icc_get_line_delay(h, &ld));
    const double calib_line_delay_us = ld * S_TO_US;
    std::cout << "g: " << g[0] << " " << g[1] << " " << g[2] << "\nT_i_c qw,qx,qy,qz: " << T[3] << " " << T[0] << " " << T[1] << " " << T[2] << "\nT_i_c t: " << T[4] << " " << T[5] << " " << T[6]
              << "\nInitialized line delay [us]: " << init_line_delay * S_TO_US << "\nCalibrated line delay [us]: " << calib_line_delay_us << "\n";
    Value out = Value::object();
    { Value q = Value::object(); q["w"] = Value(T[3]); q["x"] = Value(T[0]); q["y"] = Value(T[1]); q["z"] = Value(T[2]); out["q_i_c"] = q; }
    out["t_i_c"] = xyz(T[4], T[5], T[6]);
    out["final_reproj_error"] = Value(reproj_error);
    out["r3_dt"] = Value(ip.dt_r3_s); out["so3_dt"] = Value(ip.dt_so3_s);
    out["init_line_delay_us"] = Value(init_line_delay * S_TO_US); out["calib_line_delay_us"] = Value(calib_line_delay_us);
    out["time_offset_imu_to_cam_s"] = Value(time_offset_imu_to_cam);
    if (outlier_sigma > 0.0) { out["outlier_corners_rejected"] = Value(outliers_rejected); out["outlier_threshold_px"] = Value(outlier_threshold); }
    if (bias_walk) {
      out["bias_knot_spacing_s"] = Value(bias_dt); out["accl_random_walk"] = Value::array(); out["gyro_random_walk"] = Value::array();
      for (int a = 0; a < 3; ++a) { out["accl_random_walk"].push_back(Value(acc_q[a])); out["gyro_random_walk"].push_back(Value(gyr_q[a])); }
    }
    int n_used = 0; ICC(icc_get_num_imu_used(h, &n_used));
    std::vector<double> ut(n_used), ua(3 * (size_t)n_used), ug(3 * (size_t)n_used);
    ICC(icc_get_imu_used(h, ut.data(), ua.data(), ug.data()));
    std::vector<int64_t> t_ns(n_used); for (int i = 0; i < n_used; ++i) t_ns[i] = (int64_t)(ut[i] * S_TO_NS);
    std::vector<double> gs(3 * (size_t)n_used), as(3 * (size_t)n_used), gb(3 * (size_t)n_used), ab(3 * (size_t)n_used);
    std::vector<int32_t> valid(n_used);
    if (n_used) ICC(icc_eval_trajectory(h, n_used, t_ns.data(), gs.data(), as.data(), gb.data(), ab.data(), nullptr, nullptr, valid.data()));
    {
      CHECK_MSG(out.o->empty() || std::prev(out.o->end())->first < std::string("trajectory"), "result keys must sort before the trajectory");
      FILE* fp = fopen(F.str["result_output_json"].c_str(), "wb");
      CHECK_MSG(fp != nullptr, "could not write " << F.str["result_output_json"]);
      { iccjson::Writer w(4, fp); write_result(w, out, n_used, t_ns.data(), ug.data(), gs.data(), gb.data(), ua.data(), as.data(), ab.data()); }
      fputc('\n', fp); fclose(fp);
    }

    // ---- PLY files of the spline poses and of the input poses (app :335-364) -------------------------------------------
    std::vector<double> cam_ts(frame_t); std::sort(cam_ts.begin(), cam_ts.end());
    std::vector<int64_t> cam_ns(cam_ts.size()); for (size_t i = 0; i < cam_ts.size(); ++i) cam_ns[i] = (int64_t)(cam_ts[i] * S_TO_NS);
    std::vector<double> pq(4 * cam_ns.size()), pp(3 * cam_ns.size()); std::vector<int32_t> pvalid(cam_ns.size());
    ICC(icc_eval_trajectory(h, (int)cam_ns.size(), cam_ns.data(), nullptr, nullptr, nullptr, nullptr, pq.data(), pp.data(), pvalid.data()));
    std::vector<std::array<double, 3>> pts; std::vector<std::array<int, 3>> col;
    for (size_t i = 0; i < cam_ns.size(); ++i) {
      if (!pvalid[i]) continue;
      // T_w_c = T_w_i * T_i_c : position = p_wi + R_wi t_ic
      const double x = pq[4 * i], y = pq[4 * i + 1], z = pq[4 * i + 2], w = pq[4 * i + 3];
      const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
      pts.push_back({pp[3 * i] + R[0] * T[4] + R[1] * T[5] + R[2] * T[6], pp[3 * i + 1] + R[3] * T[4] + R[4] * T[5] + R[5] * T[6], pp[3 * i + 2] + R[6] * T[4] + R[7] * T[5] + R[8] * T[6]});
      col.push_back({0, 255, 0});
    }
    const std::string op = F.str["output_path"];
    if (!op.empty()) {
      write_ply(op + "/sparse_recon_spline.ply", pts, col);
      pts.clear(); col.clear();
      for (size_t i = 0; i < frame_t.size(); ++i) { pts.push_back({p_wc[3 * i], p_wc[3 * i + 1], p_wc[3 * i + 2]}); col.push_back({255, 0, 0}); }
      for (int i = 0; i <= max_id; ++i) { pts.push_back({board[4 * i] / board[4 * i + 3], board[4 * i + 1] / board[4 * i + 3], board[4 * i + 2] / board[4 * i + 3]}); col.push_back({255, 255, 255}); }
      write_ply(op + "/sparse_recon_calib_dataset.ply", pts, col);
    }
    icc_destroy(h);
    icc_comm_destroy(comm);        // (ncclCommDestroy waits for the peers: the rank processes are only reaped afterwards)
    for (pid_t pid : children) { int st = 0; waitpid(pid, &st, 0); if (!WIFEXITED(st) || WEXITSTATUS(st) != 0) { std::cerr << "a rank process failed" << std::endl; return 2; } }
  } catch (const std::exception& e) {
    std::cerr << "ERROR: " << e.what() << std::endl;
    return 1;
  }
  return 0;
}
