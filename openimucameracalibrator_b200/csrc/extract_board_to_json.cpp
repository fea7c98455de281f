// Drop-in host program for applications/extract_board_to_json.cc of urbste/OpenImuCameraCalibrator with --board_type radon and a folder
// of <timestamp_ns>.png frames (BoardExtractor::ExtractImageFolderToJson, src/core/board_extractor.cc): the same gflags names and
// defaults, and the same UBJSON corner file, which every other drop-in here reads.
//
// Per frame the reference runs cv::imread -> cv::resize(1/f) on the colour image -> cvtColor(BGR2GRAY) -> findChessboardCornersSB.
// Here the PNG files are decoded on the host (icc_png.hpp: the pixels imread returns) by hardware_concurrency() threads into fixed,
// index-addressed slots of two pinned batches; while one batch is on the GPU the other is being filled.  Colour frames go through
// icc_extract_radon_board_bgr (resize, then gray, as the reference orders it), gray frames through icc_extract_radon_board; a folder
// that mixes both is processed in runs of one kind.  The file depends only on the input files, never on thread timing or batch size.
//
// Refused, with a message and a non-zero exit before any output is written: --board_type other than radon (ChArUco and AprilTag
// detection are not provided; the reference treats unknown names as charuco), a regular file as --input_path (the reference's video
// route: no video decoder is available), a missing or empty folder, a file name that is not a number, a downsample factor below 1,
// a frame whose size differs from the first frame's (the reference would mix sizes under one image_width), and fewer than three
// distinct timestamps (the reference's camera_fps loop underflows there).  --aruco_detector_params and --aruco_dict are accepted and
// ignored.  --verbose prints one line per frame instead of opening a window.
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"
#include "icc_png.hpp"

#include <dirent.h>
#include <sys/stat.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <fstream>
#include <future>
#include <iostream>
#include <set>
#include <thread>

using iccjson::Value;

namespace {
using Clock = std::chrono::steady_clock;
double since(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

constexpr size_t kBatchBytes = size_t(256) << 20;   // per pinned batch; two of them

struct Frame { int channels = 0; std::string error; };

// The decoding side: frames [first, first + count) into slots of `buf`, slot_bytes apart.  A colour frame is width * 3 interleaved
// B, G, R bytes per row; a gray one width bytes per row at the same row pitch, so that every run of one kind is one strided call.
struct Decoder {
  const std::vector<std::string>& files;
  int width, height, threads;
  std::vector<Frame>& frames;
  std::vector<double> thread_seconds;
  void fill(size_t first, size_t count, uint8_t* buf) {
    std::atomic<size_t> next{0};
    const size_t row = 3 * (size_t)width, slot = row * height;
    auto work = [&](int t) {
      const auto t0 = Clock::now();
      for (size_t k; (k = next.fetch_add(1)) < count;) {
        Frame& fr = frames[first + k];
        try {
          const iccpng::Image img = iccpng::decode_file(files[first + k]);
          if (img.width != width || img.height != height)
            throw std::runtime_error(files[first + k] + ": the frame is " + std::to_string(img.width) + " x " + std::to_string(img.height) + ", the first frame " +
                                     std::to_string(width) + " x " + std::to_string(height));
          uint8_t* dst = buf + k * slot;
          const size_t n = (size_t)width * img.channels;
          if (img.channels == 3) memcpy(dst, img.px.data(), slot);
          else for (int y = 0; y < height; ++y) memcpy(dst + y * row, img.px.data() + y * n, n);
          fr.channels = img.channels;
        } catch (const std::exception& e) { fr.error = e.what(); }
      }
      thread_seconds[t] += since(t0);
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(work, t);
    work(0);
    for (auto& th : pool) th.join();
  }
};

bool is_regular_file(const std::string& p) { struct stat s; return stat(p.c_str(), &s) == 0 && S_ISREG(s.st_mode); }
bool is_directory(const std::string& p) { struct stat s; return stat(p.c_str(), &s) == 0 && S_ISDIR(s.st_mode); }

// cv::glob(dir + "/*.png", files, false) + std::sort: the non-recursive, case-sensitive *.png entries that are not directories, by full path
std::vector<std::string> png_files(const std::string& dir) {
  std::vector<std::string> out;
  DIR* d = opendir(dir.c_str());
  if (!d) return out;
  while (const dirent* e = readdir(d)) {
    const std::string name = e->d_name;
    if (name.size() < 4 || name.compare(name.size() - 4, 4, ".png") != 0) continue;
    const std::string path = dir + "/" + name;
    if (is_directory(path)) continue;
    out.push_back(path);
  }
  closedir(d);
  std::sort(out.begin(), out.end());
  return out;
}

// utils::MedianOfDoubleVec: the mean of the two middle values for an even count
double median(std::vector<double> v) {
  std::sort(v.begin(), v.end());
  const size_t n = v.size();
  return n % 2 ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) / 2;
}

Value xy(double a, double b) { Value v = Value::array(); v.push_back(Value(a)); v.push_back(Value(b)); return v; }
}  // namespace

int main(int argc, char** argv) {
  icccli::Flags F;
  F.str = {{"input_path", ""}, {"board_type", "charuco"}, {"aruco_detector_params", ""}, {"save_corners_json_path", ""}};
  F.num = {{"downsample_factor", 1.0}, {"checker_square_length_m", 0.022}, {"num_squares_x", 9}, {"num_squares_y", 7}, {"aruco_dict", 16}};
  F.boolean = {{"recompute_corners", false}, {"verbose", false}};
  try { icccli::parse_flags(argc, argv, F); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  const std::string input = F.str["input_path"], save = F.str["save_corners_json_path"];
  if (std::ifstream(save).is_open() && !F.boolean["recompute_corners"]) {
    std::cout << "Skipping corner extraction. Already extracted for: " << input << "\n";
    return 0;
  }
  const std::string type = F.str["board_type"];
  if (type != "radon") {
    std::cerr << "ERROR: --board_type " << type << " is not supported: only the radon checkerboard (--board_type radon) is detected here" << std::endl;
    return 1;
  }
  if (save.empty()) { std::cerr << "ERROR: --save_corners_json_path is empty" << std::endl; return 1; }
  if (input.empty()) { std::cerr << "ERROR: --input_path is empty" << std::endl; return 1; }
  if (is_regular_file(input)) {
    std::cerr << "ERROR: " << input << " is a file: video input is not supported, pass a folder of <timestamp_ns>.png frames" << std::endl;
    return 1;
  }
  if (!is_directory(input)) { std::cerr << "ERROR: input folder " << input << " does not exist" << std::endl; return 1; }
  const double f = F.num["downsample_factor"];
  if (!(f >= 1.0) || !std::isfinite(f)) { std::cerr << "ERROR: --downsample_factor must be a finite number >= 1, not " << f << std::endl; return 1; }
  const int W = (int)F.num["num_squares_x"], H = (int)F.num["num_squares_y"];
  const float square = (float)F.num["checker_square_length_m"];   // InitializeRadonBoard takes it as a float
  const std::vector<std::string> files = png_files(input);
  if (files.empty()) { std::cerr << "ERROR: No image files found in folder. Must be timestamp_in_ns.png!" << std::endl; return 1; }
  // timestamps from the names (std::stoul of the name after the last '/'), all before any decoding
  const size_t n = files.size();
  std::vector<int64_t> t_ns(n);
  std::set<double> timestamps_s;
  for (size_t i = 0; i < n; ++i) {
    const std::string name = files[i].substr(files[i].find_last_of('/') + 1);
    try { t_ns[i] = (int64_t)std::stoul(name); }
    catch (const std::exception&) { std::cerr << "ERROR: " << files[i] << ": the file name is not a timestamp in nanoseconds" << std::endl; return 1; }
    timestamps_s.insert(t_ns[i] * 1e-9);
  }
  if (timestamps_s.size() < 3) {
    std::cerr << "ERROR: camera_fps needs at least 3 distinct timestamps, the folder has " << timestamps_s.size() << std::endl;
    return 1;
  }
  const auto t_start = Clock::now();
  iccpng::Image first;
  try { first = iccpng::decode_file(files[0]); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  const int width = first.width, height = first.height;
  first = iccpng::Image();
  const size_t slot = (size_t)3 * width * height;
  const size_t batch = std::max<size_t>(1, std::min(n, kBatchBytes / slot));
  const int threads = (int)std::max(1u, std::thread::hardware_concurrency());
  std::cout << "Total number of frames: " << n << "\n";

  icc_handle* h = nullptr;
  icc_status st = icc_create(&h, 0);
  if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
  void* bufs[2] = {nullptr, nullptr};
  for (void*& b : bufs)
    if ((st = icc_host_alloc_pinned(slot * batch, &b)) != ICC_OK) {
      std::cerr << "could not allocate " << slot * batch << " bytes of pinned host memory (" << st << ")" << std::endl;
      icc_host_free_pinned(bufs[0]); icc_destroy(h); return 2;
    }
  std::vector<Frame> frames(n);
  Decoder D{files, width, height, threads, frames, std::vector<double>(threads, 0.0)};
  const size_t per = (size_t)W * H;
  std::vector<double> uv(n * per * 2, 0.0);
  std::vector<int32_t> found(n, 0);
  int out_w = 0, out_h = 0;
  double gpu_seconds = 0.0;
  int rc = 0;
  const size_t n_batches = (n + batch - 1) / batch;
  std::future<void> pending = std::async(std::launch::async, [&] { D.fill(0, std::min(batch, n), (uint8_t*)bufs[0]); });
  for (size_t b = 0; b < n_batches && rc == 0; ++b) {
    pending.get();
    const size_t first_i = b * batch, count = std::min(batch, n - first_i);
    if (b + 1 < n_batches)
      pending = std::async(std::launch::async, [&, b] { D.fill((b + 1) * batch, std::min(batch, n - (b + 1) * batch), (uint8_t*)bufs[(b + 1) % 2]); });
    for (size_t k = 0; k < count; ++k)
      if (!frames[first_i + k].error.empty()) { std::cerr << "ERROR: " << frames[first_i + k].error << std::endl; rc = 1; break; }
    if (rc) break;
    const uint8_t* buf = (const uint8_t*)bufs[b % 2];
    for (size_t k0 = 0; k0 < count;) {   // runs of one kind
      size_t k1 = k0 + 1;
      const int ch = frames[first_i + k0].channels;
      while (k1 < count && frames[first_i + k1].channels == ch) ++k1;
      icc_board_summary S;
      const size_t i0 = first_i + k0;
      st = (ch == 3 ? icc_extract_radon_board_bgr : icc_extract_radon_board)(h, (int)(k1 - k0), width, height, 3 * (int64_t)width, buf + k0 * slot, W, H, f,
                                                                          uv.data() + i0 * per * 2, found.data() + i0, &S);
      if (st != ICC_OK) { std::cerr << "board extraction failed (" << st << "): " << icc_last_error(h) << std::endl; rc = 2; break; }
      out_w = S.width; out_h = S.height; gpu_seconds += S.seconds;
      k0 = k1;
    }
    if (rc) break;
    for (size_t k = 0; k < count; ++k) {
      const size_t i = first_i + k;
      if (F.boolean["verbose"]) std::cout << files[i] << ": " << (found[i] ? std::to_string(per) + " corners" : std::string("board not found")) << "\n";
      if ((i + 1) % 60 == 0) std::cout << "Extracting corners from frame " << i + 1 << " / " << n << "\n";
    }
  }
  if (pending.valid()) pending.wait();
  icc_host_free_pinned(bufs[0]); icc_host_free_pinned(bufs[1]);
  icc_destroy(h);
  if (rc) return rc;

  // the corner file, as nlohmann::json::to_ubjson writes the reference's document
  Value doc = Value::object();
  doc["calibration_board_type"] = Value(1);                      // BoardType::RADON
  doc["square_size_meter"] = Value((double)square);
  Value pts = Value::array();                                    // output_json["scene_pts"][int id]: an array indexed by id
  for (int i = 0; i < H; ++i)
    for (int j = 0; j < W; ++j) {                                // cv::Point3f((float)i * s, (float)j * s, 0.f)
      Value p = Value::array();
      p.push_back(Value((double)((float)i * square))); p.push_back(Value((double)((float)j * square))); p.push_back(Value(0.0));
      pts.push_back(p);
    }
  doc["scene_pts"] = pts;
  doc["image_width"] = Value(out_w); doc["image_height"] = Value(out_h);
  int n_found = 0;
  for (size_t i = 0; i < n; ++i) {
    if (!found[i]) continue;
    ++n_found;
    const double timestamp_s = t_ns[i] * 1e-9;
    Value& ip = doc["views"][std::to_string(timestamp_s * 1e6)]["image_points"];
    for (size_t c = 0; c < per; ++c) ip[std::to_string(c)] = xy(uv[(i * per + c) * 2], uv[(i * per + c) * 2 + 1]);
  }
  const std::vector<double> times(timestamps_s.begin(), timestamps_s.end());
  std::vector<double> dt;
  for (size_t i = 0; i < times.size() - 2; ++i) dt.push_back(times[i + 1] - times[i]);   // the reference's bound: the last interval is not used
  doc["camera_fps"] = Value(1.0 / median(dt));
  const std::string bytes = iccjson::dump_ubjson(doc);
  std::ofstream out(save, std::ios::out | std::ios::binary);
  out.write(bytes.data(), (std::streamsize)bytes.size());
  out.close();
  if (!out) { std::cerr << "ERROR: could not write " << save << std::endl; return 1; }
  double decode_seconds = 0.0;
  for (double s : D.thread_seconds) decode_seconds += s;
  std::cout << "Found the board in " << n_found << " of " << n << " frames; wall " << since(t_start) << " s, decode " << decode_seconds << " s summed over "
            << threads << " threads, GPU " << gpu_seconds << " s\n";
  return 0;
}
