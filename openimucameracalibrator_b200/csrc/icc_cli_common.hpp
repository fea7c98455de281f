// Pieces shared by the drop-in command line tools: gflags-style parsing, the camera calibration JSON reader and the corner file
// (scene) reader.  Header-only, host C++.
#pragma once
#include "../../include/icc_b200.h"
#include "icc_json.hpp"

#include <algorithm>
#include <cstdint>
#include <map>
#include <ostream>
#include <stdexcept>
#include <cmath>
#include <string>
#include <utility>
#include <vector>

namespace icccli {
using iccjson::Value;

struct Flags {   // every tool fills in its own names and defaults
  std::map<std::string, std::string> str;
  std::map<std::string, bool> boolean;
  std::map<std::string, double> num;
};

// --pose_error of the pose tools: the residual of the per-view pose step (icc_set_pose_error); any other value is a usage error
inline int parse_pose_error(const std::string& v) {
  if (v == "normalized") return ICC_POSE_ERROR_NORMALIZED;
  if (v == "tangent") return ICC_POSE_ERROR_TANGENT;
  throw std::runtime_error("flag --pose_error must be 'normalized' or 'tangent', not '" + v + "'");
}

// --reprojection_error of the hot CLI: the vision residual of the spline solve (icc_set_reprojection_error); any other value is a usage error
inline int parse_reprojection_error(const std::string& v) {
  if (v == "pixel") return ICC_REPROJ_ERROR_PIXEL;
  if (v == "tangent") return ICC_REPROJ_ERROR_TANGENT;
  throw std::runtime_error("flag --reprojection_error must be 'pixel' or 'tangent', not '" + v + "'");
}

// --pose_shutter of the pose tools: true = rolling (icc_set_pose_rolling_shutter); any other value than global / rolling is a usage error
inline bool parse_pose_shutter(const std::string& v) {
  if (v == "global") return false;
  if (v == "rolling") return true;
  throw std::runtime_error("flag --pose_shutter must be 'global' or 'rolling', not '" + v + "'");
}

// the line delay of --pose_shutter rolling: one readout per frame interval, 1 / fps / image height (the hot CLI's initial line delay)
inline double pose_line_delay(double fps, int height) {
  if (!(fps > 0.0) || height <= 0) throw std::runtime_error("--pose_shutter rolling needs fps > 0 and an image height in the camera calibration");
  return 1.0 / fps / height;
}

// Random-walk densities in Kalibr's units (m/s^3/sqrt(Hz), rad/s^2/sqrt(Hz)) from a fit_allan_variance --output_json document: per axis
// q = sqrt(3) |K| / scale, K the channel's fitted rate-random-walk term, scale 1 for the accelerometer (m/s^2) and 57.3 * 3600 for the
// gyroscope (deg/h).  The Python statement is io_formats.bias_random_walk_from_allan.
inline void bias_random_walk_from_allan(const Value& doc, double acc_q[3], double gyr_q[3]) {
  const char* axes[3] = {"x", "y", "z"};
  for (int a = 0; a < 3; ++a) {
    acc_q[a] = std::sqrt(3.0) * std::fabs(doc.at("channels").at(std::string("acc_") + axes[a]).at("params").at("K").num()) / 1.0;
    gyr_q[a] = std::sqrt(3.0) * std::fabs(doc.at("channels").at(std::string("gyr_") + axes[a]).at("params").at("K").num()) / (57.3 * 3600);
  }
}

inline bool parse_bool(const std::string& v) { return v == "true" || v == "1" || v == "t" || v == "yes" || v == "y" || v == "True"; }

// gflags syntax: --name=value, --name value, -name..., --boolflag, --noboolflag
inline void parse_flags(int argc, char** argv, Flags& f) {
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    if (a.size() < 2 || a[0] != '-') throw std::runtime_error("unexpected argument: " + a);
    a = a.substr(a[1] == '-' ? 2 : 1);
    std::string name = a, value; bool has_value = false;
    const size_t eq = a.find('=');
    if (eq != std::string::npos) { name = a.substr(0, eq); value = a.substr(eq + 1); has_value = true; }
    if (f.boolean.count(name)) { f.boolean[name] = has_value ? parse_bool(value) : true; continue; }
    if (name.rfind("no", 0) == 0 && f.boolean.count(name.substr(2)) && !has_value) { f.boolean[name.substr(2)] = false; continue; }
    if (!has_value) { if (i + 1 >= argc) throw std::runtime_error("flag --" + name + " needs a value"); value = argv[++i]; }
    if (f.str.count(name)) f.str[name] = value;
    else if (f.num.count(name)) f.num[name] = std::stod(value);
    else throw std::runtime_error("unknown command line flag '" + name + "'");
  }
}


// The camera JSON (src/io/read_camera_calibration.cc:35-119, src/io/write_camera_calibration.cc:33-133) and the model line of
// CameraCalibrator::PrintResult (src/core/camera_calibrator.cc:391-458), one row per model.  The same table, row for row, is CAMERAS in
// openimucameracalibrator_b200/camera_models.py.
using CameraKeys = std::vector<std::pair<std::string, int>>;
struct CameraLayout {
  std::string name;     // `intrinsic_type`, --camera_model_to_calibrate
  int id, num_params;
  CameraKeys keys;      // (JSON key, Theia index) of every intrinsic the file carries; `skew` only where index 2 is the skew
  CameraKeys printed;   // (label, index) of the model's PrintResult line, "" for an unlabelled value; empty when the tools print none
  int index(const std::string& key) const { for (const auto& [k, i] : keys) if (k == key) return i; throw std::runtime_error("no intrinsic " + key); }
};
inline CameraKeys affine_keys(bool skew, CameraKeys own) {   // focal length, aspect ratio, [skew,] principal point, then the model's own keys
  CameraKeys k = skew ? CameraKeys{{"focal_length", 0}, {"aspect_ratio", 1}, {"skew", 2}, {"principal_pt_x", 3}, {"principal_pt_y", 4}}
                      : CameraKeys{{"focal_length", 0}, {"aspect_ratio", 1}, {"principal_pt_x", 2}, {"principal_pt_y", 3}};
  k.insert(k.end(), own.begin(), own.end());
  return k;
}
inline const std::vector<CameraLayout> kCameraLayouts = {
  {"PINHOLE", ICC_CAM_PINHOLE, 7, affine_keys(true, {}), {}},
  {"PINHOLE_RADIAL_TANGENTIAL", ICC_CAM_PINHOLE_RADIAL_TANGENTIAL, 10,
   affine_keys(true, {{"radial_distortion_1", 5}, {"radial_distortion_2", 6}, {"radial_distortion_3", 7}, {"tangential_distortion_1", 8}, {"tangential_distortion_2", 9}}), {}},
  {"FISHEYE", ICC_CAM_FISHEYE, 9, affine_keys(true, {{"radial_distortion_1", 5}, {"radial_distortion_2", 6}, {"radial_distortion_3", 7}, {"radial_distortion_4", 8}}),
   {{"Radial distortion 1", 5}, {"Radial distortion 2", 6}, {"Radial distortion 3", 7}, {"Radial distortion 4", 8}}},
  {"FOV", ICC_CAM_FOV, 5, affine_keys(false, {{"radial_distortion_1", 4}}), {}},
  {"DIVISION_UNDISTORTION", ICC_CAM_DIVISION_UNDISTORTION, 5, affine_keys(false, {{"div_undist_distortion", 4}}), {{"Distortion", 4}}},
  {"DOUBLE_SPHERE", ICC_CAM_DOUBLE_SPHERE, 7, affine_keys(true, {{"xi", 5}, {"alpha", 6}}), {{"XI", 5}, {"ALPHA", 6}}},
  {"EXTENDED_UNIFIED", ICC_CAM_EXTENDED_UNIFIED, 7, affine_keys(true, {{"alpha", 5}, {"beta", 6}}), {{"", 5}, {"BETA", 6}}},
  {"OMNI_RADIAL_TANGENTIAL", ICC_CAM_OMNI_RADIAL_TANGENTIAL, 10,
   affine_keys(true, {{"xi", 5}, {"radial_distortion_1", 6}, {"radial_distortion_2", 7}, {"tangential_distortion_1", 8}, {"tangential_distortion_2", 9}}),
   {{"XI", 5}, {"Radial distortion 1", 6}, {"Radial distortion 2", 7}, {"Tangential distortion 1", 8}, {"Tangential distortion 2", 9}}},
  {"SCARAMUZZA", ICC_CAM_SCARAMUZZA, 9,   // index 2 is the stretch e, not a skew
   {{"focal_length", 0}, {"aspect_ratio", 1}, {"principal_pt_x", 3}, {"principal_pt_y", 4}, {"stretch_d", 8}, {"stretch_e", 2}, {"polynomial_a2", 5}, {"polynomial_a3", 6}, {"polynomial_a4", 7}},
   {{"A2", 5}, {"A3", 6}, {"A4", 7}, {"Stretch c", 1}, {"d", 8}, {"e", 2}}},
  {"PINHOLE_RATIONAL", ICC_CAM_PINHOLE_RATIONAL, 13,
   affine_keys(true, {{"radial_distortion_1", 5}, {"radial_distortion_2", 6}, {"radial_distortion_3", 7}, {"tangential_distortion_1", 8}, {"tangential_distortion_2", 9},
                      {"radial_distortion_4", 10}, {"radial_distortion_5", 11}, {"radial_distortion_6", 12}}),
   {{"Radial distortion 1", 5}, {"Radial distortion 2", 6}, {"Radial distortion 3", 7}, {"Radial distortion 4", 10}, {"Radial distortion 5", 11}, {"Radial distortion 6", 12},
    {"Tangential distortion 1", 8}, {"Tangential distortion 2", 9}}},
  {"FISHEYE_RADIAL_TANGENTIAL", ICC_CAM_FISHEYE_RADIAL_TANGENTIAL, 13,
   affine_keys(true, {{"radial_distortion_1", 5}, {"radial_distortion_2", 6}, {"radial_distortion_3", 7}, {"radial_distortion_4", 8}, {"radial_distortion_5", 9},
                      {"radial_distortion_6", 10}, {"tangential_distortion_1", 11}, {"tangential_distortion_2", 12}}),
   {{"Radial distortion 1", 5}, {"Radial distortion 2", 6}, {"Radial distortion 3", 7}, {"Radial distortion 4", 8}, {"Radial distortion 5", 9}, {"Radial distortion 6", 10},
    {"Tangential distortion 1", 11}, {"Tangential distortion 2", 12}}},
};

// theia::StringToCameraIntrinsicsModelType: the row of a model name, nullptr for an unknown one
inline const CameraLayout* find_camera(const std::string& name) {
  for (const CameraLayout& c : kCameraLayouts) if (c.name == name) return &c;
  return nullptr;
}

// camera JSON -> (model id, Theia-ordered intrinsics).  Like the reference, `skew` is never read; FOV's aspect_ratio may be absent (1.0).
inline int read_camera(const Value& j, std::vector<double>& k, int& width, int& height, double& fps) {
  const std::string type = j.at("intrinsic_type").str();
  const Value& in = j.at("intrinsics");
  width = (int)j.at("image_width").num(); height = (int)j.at("image_height").num(); fps = j.at("fps").num();
  const CameraLayout* c = find_camera(type);
  if (!c) throw std::runtime_error("unknown intrinsic_type " + type);
  k.assign(c->num_params, 0.0);
  for (const auto& [key, i] : c->keys) {
    if (key == "skew") continue;
    k[i] = c->id == ICC_CAM_FOV && key == "aspect_ratio" && !in.contains(key) ? 1.0 : in.at(key).num();
  }
  return c->id;
}

// the `intrinsics` object of the camera JSON: every key of the layout, and `skew` 0 for the models whose index 2 is no skew
inline Value write_intrinsics(const CameraLayout& c, const double* k) {
  Value in = Value::object();
  in["skew"] = Value(0.0);
  for (const auto& [key, i] : c.keys) in[key] = Value(k[i]);
  return in;
}

// CameraCalibrator::PrintResult: the focal length and principal point line, then the model's line if it has one
inline void print_camera(std::ostream& os, const CameraLayout& c, const double* k) {
  os << "Focal Length:" << k[0] << "px Principal Point: " << k[c.index("principal_pt_x")] << "/" << k[c.index("principal_pt_y")] << "px.\n";
  if (c.printed.empty()) return;
  os << c.name << " model:";
  for (const auto& [label, i] : c.printed) os << " " << label << (label.empty() ? "" : ": ") << k[i];
  os << "\n";
}

// Corner file (src/core/board_extractor.cc:294-296,325-333,375-380): scene_pts {"id": [x,y,z]} -> homogeneous board points by id.
// The reference writes the radon board's points with an integer index, so there scene_pts is an array [[x,y,z], ...] whose index is the
// id; read_scene.cc iterates items(), which takes either form, and so does this.
inline std::vector<double> read_scene_points(const Value& scene_json, int& n_points) {
  const Value& pts = scene_json.at("scene_pts");
  if (pts.is_array()) {
    const int n = (int)pts.size();
    std::vector<double> board(4 * (size_t)n, 0.0);
    for (int id = 0; id < n; ++id) { for (int d = 0; d < 3; ++d) board[4 * id + d] = pts.at(id).at(d).num(); board[4 * id + 3] = 1.0; }
    n_points = n;
    return board;
  }
  if (!pts.is_object()) throw std::runtime_error("scene_pts must be an object or an array");
  int max_id = -1; for (const auto& kv : *pts.o) max_id = std::max(max_id, std::stoi(kv.first));
  std::vector<double> board(4 * (size_t)(max_id + 1), 0.0);
  for (int i = 0; i <= max_id; ++i) board[4 * i + 3] = 1.0;
  for (const auto& kv : *pts.o) { const int id = std::stoi(kv.first); for (int d = 0; d < 3; ++d) board[4 * id + d] = kv.second.at(d).num(); }
  n_points = max_id + 1;
  return board;
}

// Views of the corner file in std::map key order (what nlohmann::json iteration gives the reference): the key as written, the
// timestamp [us] it spells, CSR corner lists with the ids of a view in lexicographic order of their decimal strings.
struct SceneViews { std::vector<std::string> key; std::vector<double> timestamp_us; std::vector<int32_t> off{0}, ids; std::vector<double> uv; };
inline SceneViews read_scene_views(const Value& scene_json) {
  SceneViews v;
  for (const auto& kv : *scene_json.at("views").o) {
    v.key.push_back(kv.first); v.timestamp_us.push_back(std::stod(kv.first));
    for (const auto& ip : *kv.second.at("image_points").o) { v.ids.push_back(std::stoi(ip.first)); v.uv.push_back(ip.second.at(0).num()); v.uv.push_back(ip.second.at(1).num()); }
    v.off.push_back((int32_t)v.ids.size());
  }
  return v;
}

// Streaming reader of the corner file: the "views" member -- hundreds of thousands of tiny nested objects, > 95 % of the file -- goes
// straight into the CSR arrays (same order and same last-duplicate-wins rule as the std::map route above), every other member is
// returned as a Value.  Any structural surprise throws; load_scene() then falls back to the generic route.
class SceneUbjsonReader : public iccjson::UbjsonParser {
 public:
  using iccjson::UbjsonParser::UbjsonParser;
  Value parse_scene(SceneViews& sv) {
    if (next() != '{') fail("expected an object");
    Value meta = Value::object(); bool have_views = false;
    members([&](std::string& key, unsigned char t) {
      if (key == "views" && t == '{') { parse_views(sv); have_views = true; }
      else meta.o->insert_or_assign(std::move(key), value(t));
    });
    if (!have_views) fail("no views object");
    return meta;
  }
 private:
  void header(unsigned char& et, int64_t& n) {
    et = 0; n = -1;
    if (peek() == '$') { ++p_; et = next(); if (next() != '#') fail("expected '#' after '$'"); n = integer(next()); }
    else if (peek() == '#') { ++p_; n = integer(next()); }
  }
  template <class F> void members(F f) {     // after '{'; f consumes exactly the value whose type marker it is handed
    unsigned char et; int64_t n; header(et, n);
    if (n >= 0) { for (int64_t k = 0; k < n; ++k) { std::string key = raw_string(); f(key, et ? et : next()); } }
    else { while (peek() != '}') { std::string key = raw_string(); f(key, next()); } ++p_; }
  }
  template <class F> void elements(F f) {    // after '['
    unsigned char et; int64_t n; header(et, n);
    if (n >= 0) { for (int64_t k = 0; k < n; ++k) f(et ? et : next()); }
    else { while (peek() != ']') f(next()); ++p_; }
  }
  double number(unsigned char t) {
    switch (t) {
      case 'i': case 'U': case 'I': case 'l': case 'L': case 'u': case 'm': case 'M': return (double)integer(t);
      case 'd': return (double)be<float>(); case 'D': return be<double>();
      case 'H': return std::stod(raw_string());
      default: fail("expected a number");
    }
  }
  struct Corner { std::string id; double u, v; };
  struct View { std::string key; std::vector<Corner> corners; };
  void parse_views(SceneViews& sv) {
    std::vector<View> views;
    members([&](std::string& key, unsigned char t) {
      if (t != '{') fail("a view must be an object");
      View vw; vw.key = std::move(key); bool have_points = false;
      members([&](std::string& k2, unsigned char t2) {
        if (k2 == "image_points" && t2 == '{') {
          have_points = true;
          members([&](std::string& id, unsigned char t3) {
            if (t3 != '[') fail("an image point must be an array");
            double xy[2] = {0.0, 0.0}; int c = 0;
            elements([&](unsigned char t4) { const double x = number(t4); if (c < 2) xy[c] = x; ++c; });
            if (c < 2) fail("an image point needs two coordinates");
            vw.corners.push_back({std::move(id), xy[0], xy[1]});
          });
        } else (void)value(t2);
      });
      if (!have_points) fail("view without image_points");
      views.push_back(std::move(vw));
    });
    // std::map semantics: keys in lexicographic order, a repeated key keeps its last value
    std::stable_sort(views.begin(), views.end(), [](const View& a, const View& b) { return a.key < b.key; });
    for (size_t i = 0; i < views.size(); ++i) {
      if (i + 1 < views.size() && views[i + 1].key == views[i].key) continue;
      View& vw = views[i];
      std::stable_sort(vw.corners.begin(), vw.corners.end(), [](const Corner& a, const Corner& b) { return a.id < b.id; });
      sv.key.push_back(vw.key); sv.timestamp_us.push_back(std::stod(vw.key));
      for (size_t c = 0; c < vw.corners.size(); ++c) {
        if (c + 1 < vw.corners.size() && vw.corners[c + 1].id == vw.corners[c].id) continue;
        sv.ids.push_back(std::stoi(vw.corners[c].id)); sv.uv.push_back(vw.corners[c].u); sv.uv.push_back(vw.corners[c].v);
      }
      sv.off.push_back((int32_t)sv.ids.size());
    }
  }
};
// corner file -> (every member but "views", the views); scene_json stays usable with read_scene_points / at("image_width") ...
inline Value load_scene(const std::string& path, SceneViews& sv) {
  const std::string data = iccjson::read_file(path, true);
  try { SceneViews fast; Value meta = SceneUbjsonReader(data).parse_scene(fast); sv = std::move(fast); return meta; }
  catch (const std::exception&) { }
  Value doc = iccjson::UbjsonParser(data).parse();    // generic route: reports malformed files with the usual messages
  sv = read_scene_views(doc);
  return doc;
}

// Telemetry JSON (src/io/read_telemetry.cc:29-69): the three long arrays are read straight into flat vectors, everything else into `meta`.
struct Telemetry { std::vector<double> t_ns, acc, gyr, img_t_ns; Value meta; };
class TelemetryReader : public iccjson::TextParser {
 public:
  using iccjson::TextParser::TextParser;
  void parse_telemetry(Telemetry& T) {
    T.meta = Value::object();
    ws(); if (p_ >= t_.size() || t_[p_] != '{') fail("expected an object");
    ++p_; ws();
    if (p_ < t_.size() && t_[p_] == '}') { ++p_; return; }
    for (;;) {
      ws(); if (p_ >= t_.size() || t_[p_] != '"') fail("expected key");
      std::string k = string(); ws();
      if (p_ >= t_.size() || t_[p_] != ':') fail("expected ':'");
      ++p_; ws();
      if (k == "accelerometer") { T.acc.clear(); triples(T.acc); }
      else if (k == "gyroscope") { T.gyr.clear(); triples(T.gyr); }
      else if (k == "timestamps_ns") { T.t_ns.clear(); numbers(T.t_ns); }
      else if (k == "img_timestamps_ns") { T.img_t_ns.clear(); numbers(T.img_t_ns); }
      else T.meta.o->insert_or_assign(std::move(k), value());
      ws();
      if (p_ < t_.size() && t_[p_] == ',') { ++p_; continue; }
      if (p_ < t_.size() && t_[p_] == '}') { ++p_; break; }
      fail("expected ',' or '}'");
    }
    ws(); if (p_ != t_.size()) fail("trailing characters");
  }
 private:
  template <class F> void array(F f) {
    if (p_ >= t_.size() || t_[p_] != '[') fail("expected an array");
    ++p_; ws();
    if (p_ < t_.size() && t_[p_] == ']') { ++p_; return; }
    for (;;) {
      ws(); f(); ws();
      if (p_ < t_.size() && t_[p_] == ',') { ++p_; continue; }
      if (p_ < t_.size() && t_[p_] == ']') { ++p_; return; }
      fail("expected ',' or ']'");
    }
  }
  void numbers(std::vector<double>& out) { array([&]() { out.push_back(number().num()); }); }
  void triples(std::vector<double>& out) {
    array([&]() { int c = 0; array([&]() { const double v = number().num(); if (c < 3) out.push_back(v); ++c; }); if (c < 3) fail("a sample needs three components"); });
  }
};
inline Telemetry load_telemetry(const std::string& path) {
  const std::string text = iccjson::read_file(path);
  Telemetry T;
  try { TelemetryReader(text).parse_telemetry(T); return T; } catch (const std::exception&) { }
  // generic route (also the one that reports malformed files)
  Telemetry G; G.meta = iccjson::parse_text(text);
  auto flat = [&](const char* key, std::vector<double>& out, int dim) {
    if (!G.meta.contains(key)) return;
    const Value& a = G.meta.at(key);
    for (size_t i = 0; i < a.size(); ++i) { if (dim == 1) out.push_back(a.at(i).num()); else for (int d = 0; d < dim; ++d) out.push_back(a.at(i).at(d).num()); }
  };
  (void)G.meta.at("timestamps_ns"); (void)G.meta.at("gyroscope");   // missing streams are reported by name
  flat("timestamps_ns", G.t_ns, 1); flat("accelerometer", G.acc, 3); flat("gyroscope", G.gyr, 3); flat("img_timestamps_ns", G.img_t_ns, 1);
  return G;
}
// view name in the pose dataset: std::to_string((uint64_t)(timestamp_s * S_TO_US)) with timestamp_s = timestamp_us * US_TO_S (pose_estimator.cc:119-120,146)
inline std::string pose_view_name(double timestamp_us) { const double timestamp_s = timestamp_us * 1e-6; return std::to_string((uint64_t)(timestamp_s * 1e6)); }

}  // namespace icccli
