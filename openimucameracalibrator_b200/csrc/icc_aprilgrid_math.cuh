// Per-tag and per-corner math of the AprilGrid extraction (icc_aprilgrid.cu), kept in a header so that
// tests/board/aprilgrid_host_math.cu compiles exactly this code for the CPU.
//
// Reference: BoardExtractor::ExtractBoard with BoardType::APRILTAG (src/core/board_extractor.cc), i.e. the Kalibr/Basalt wrapper
// ApriltagDetector::detectTags (third_party/apriltag/apriltag.cpp) around the ethz AprilTags detector (TagDetector.cc, TagFamily.cc).
// Conventions (DESIGN.md "AprilGrid corners"):
//   - the quad frame: corners q0..q3 in image pixels (centres at integer coordinates) with a negative shoelace sum, which is
//     bottom-left, bottom-right, top-right, top-left of a board seen from the front with its y axis up; (x, y) in [0, 1]^2 maps to
//     the quad by the projective map with (0, 0) -> q0, (1, 0) -> q1, (1, 1) -> q2, (0, 1) -> q3;
//   - a tag is 10 x 10 cells (a 2-cell black border around 6 x 6 data cells); the code is read from data row iy = 5 down to 0,
//     column 0 to 5, the first bit the most significant, bit 1 where the pixel is brighter than the mean of a black and a white
//     bilinear model (TagDetector.cc, step eight);
//   - the decoded tag's bottom-left corner is q[rot], where rot is the number of quarter turns rotate90 applied to the read code.
#pragma once
#include "icc_device_math.cuh"
#include "icc_tag36h11.h"

#include <cmath>
#include <cstdint>

namespace icc {
namespace aprilgrid {

constexpr int kDim = 6, kBlackBorder = 2, kCells = kDim + 2 * kBlackBorder;   // 10 x 10 cells
constexpr int kErrorRecoveryBits = 1;        // TagFamily::errorRecoveryBits: good iff the Hamming distance is <= 1
constexpr double kMinBorderDistance = 4.0;   // px; ApriltagDetectorData::minBorderDistance
constexpr int kMinTags = 4;                  // minTagsForValidObs
// ApriltagDetectorData::size() is 36 * 4 whatever the board, so the wrapper drops every id >= 36 / ... = 36 * 4 / 4 on any board
constexpr int kIdLimit = 36;
constexpr int kSubpixMaxIters = 100;         // cv::TermCriteria(EPS + MAX_ITER, 100, 0.01)
constexpr double kSubpixEps = 0.01;

// ---- the quad's projective map (Heckbert's unit square to quadrilateral), FP64 ------------------------------------------------
struct QuadMap { double a, b, c, d, e, f, g, h; };

ICC_HD QuadMap quad_map(const double q[8]) {
  const double x0 = q[0], y0 = q[1], x1 = q[2], y1 = q[3], x2 = q[4], y2 = q[5], x3 = q[6], y3 = q[7];
  const double sx = x0 - x1 + x2 - x3, sy = y0 - y1 + y2 - y3;
  const double dx1 = x1 - x2, dx2 = x3 - x2, dy1 = y1 - y2, dy2 = y3 - y2;
  const double den = dx1 * dy2 - dx2 * dy1;
  QuadMap m;
  m.g = (sx * dy2 - dx2 * sy) / den;
  m.h = (dx1 * sy - sx * dy1) / den;
  m.a = x1 - x0 + m.g * x1; m.b = x3 - x0 + m.h * x3; m.c = x0;
  m.d = y1 - y0 + m.g * y1; m.e = y3 - y0 + m.h * y3; m.f = y0;
  return m;
}

ICC_HD void quad_apply(const QuadMap& m, double x, double y, double& px, double& py) {
  const double z = m.g * x + m.h * y + 1.0;
  px = (m.a * x + m.b * y + m.c) / z;
  py = (m.d * x + m.e * y + m.f) / z;
}

// ---- sampling the tag -------------------------------------------------------------------------------------------------------
// The 12 x 12 sample positions (ix, iy) = -1 .. kCells of the grey models, k = (iy + 1) 12 + ix + 1; the white model takes the ring
// just outside the tag, the black model the tag's outermost ring, the rest are not used (kind 0).
constexpr int kModelSamples = (kCells + 2) * (kCells + 2);
ICC_HD int model_kind(int k, int& ix, int& iy) {
  ix = k % (kCells + 2) - 1; iy = k / (kCells + 2) - 1;
  if (iy == -1 || iy == kCells || ix == -1 || ix == kCells) return 2;        // white
  if (iy == 0 || iy == kCells - 1 || ix == 0 || ix == kCells - 1) return 1;  // black
  return 0;
}

// the pixel the detector reads at quad coordinates (x, y): (int)(p + 0.5), as TagDetector.cc does (truncation); false outside
ICC_HD bool sample_pixel(const uint8_t* img, int64_t pitch, int w, int h, const QuadMap& m, double x, double y, double& v) {
  double px, py;
  quad_apply(m, x, y, px, py);
  const int irx = (int)(px + 0.5), iry = (int)(py + 0.5);
  if (irx < 0 || irx >= w || iry < 0 || iry >= h) return false;
  v = (double)img[(int64_t)iry * pitch + irx];
  return true;
}

// GrayModel: least squares of v = c0 x + c1 y + c2 x y + c3; s = {A00, A01, A02, A03, A11, A12, A13, A22, A23, A33, b0, b1, b2, b3, n}
constexpr int kGraySums = 15;
ICC_HD void gray_add(double s[kGraySums], double x, double y, double v) {
  const double xy = x * y;
  s[0] += x * x; s[1] += x * y; s[2] += x * xy; s[3] += x;
  s[4] += y * y; s[5] += y * xy; s[6] += y;
  s[7] += xy * xy; s[8] += xy; s[9] += 1.0;
  s[10] += x * v; s[11] += y * v; s[12] += xy * v; s[13] += v; s[14] += 1.0;
}

// the model's coefficients; with fewer than 6 observations or a singular system the constant model (the mean), as GrayModel::compute
ICC_HD void gray_solve(const double s[kGraySums], double c[4]) {
  c[0] = c[1] = c[2] = 0.0; c[3] = s[14] > 0 ? s[13] / s[14] : 0.0;
  if (s[14] < 6) return;
  double A[4][5] = {{s[0], s[1], s[2], s[3], s[10]}, {s[1], s[4], s[5], s[6], s[11]}, {s[2], s[5], s[7], s[8], s[12]}, {s[3], s[6], s[8], s[9], s[13]}};
  for (int k = 0; k < 4; ++k) {
    int p = k;
    for (int r = k + 1; r < 4; ++r) if (fabs(A[r][k]) > fabs(A[p][k])) p = r;
    if (!(fabs(A[p][k]) > 1e-12 * (fabs(A[0][0]) + fabs(A[3][3])))) { c[0] = c[1] = c[2] = 0.0; c[3] = s[13] / s[14]; return; }
    if (p != k) for (int j = 0; j < 5; ++j) { const double t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
    for (int r = k + 1; r < 4; ++r) {
      const double f = A[r][k] / A[k][k];
      for (int j = k; j < 5; ++j) A[r][j] -= f * A[k][j];
    }
  }
  double x[4];
  for (int k = 3; k >= 0; --k) {
    double t = A[k][4];
    for (int j = k + 1; j < 4; ++j) t -= A[k][j] * x[j];
    x[k] = t / A[k][k];
  }
  for (int k = 0; k < 4; ++k) c[k] = x[k];
}

ICC_HD double gray_eval(const double c[4], double x, double y) { return c[0] * x + c[1] * y + c[2] * x * y + c[3]; }

// data bit k = 0 .. 35 in reading order (k = 0 is the most significant): its quad coordinates
ICC_HD void bit_position(int k, double& x, double& y) {
  const int iy = kDim - 1 - k / kDim, ix = k % kDim;
  x = (kBlackBorder + ix + 0.5) / kCells;
  y = (kBlackBorder + iy + 0.5) / kCells;
}

// TagFamily::rotate90: one quarter turn of a d x d code (clockwise with y up)
ICC_HD uint64_t rotate90(uint64_t w) {
  uint64_t r = 0;
  for (int row = kDim - 1; row >= 0; --row)
    for (int col = 0; col < kDim; ++col) r = (r << 1) | ((w >> (row + kDim * col)) & 1ull);
  return r;
}

ICC_HD int popcount64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __popcll(x);
#else
  return __builtin_popcountll(x);
#endif
}

// TagFamily::decode over codes[first], codes[first + stride], ...: the smallest (Hamming distance, id, rotation), packed as
// key = (distance * kTag36h11Count + id) * 4 + rot so that the minimum key is the reference's choice (first strictly better)
ICC_HD int decode_key(uint64_t code, const uint64_t* codes, int first, int stride) {
  uint64_t r[4];
  r[0] = code; r[1] = rotate90(r[0]); r[2] = rotate90(r[1]); r[3] = rotate90(r[2]);
  int best = 0x7fffffff;
  for (int id = first; id < kTag36h11Count; id += stride)
    for (int rot = 0; rot < 4; ++rot) {
      const int key = (popcount64(r[rot] ^ codes[id]) * kTag36h11Count + id) * 4 + rot;
      best = key < best ? key : best;
    }
  return best;
}
ICC_HD void unpack_key(int key, int& hamming, int& id, int& rot) { rot = key & 3; id = (key >> 2) % kTag36h11Count; hamming = (key >> 2) / kTag36h11Count; }

// ---- the wrapper's rules for one frame (ApriltagDetector::detectTags) -------------------------------------------------------------
// p: the tag's corners (x, y) x 4 in the detector's order; the border test compares floats, as the wrapper does
ICC_HD bool near_border(const double p[8], int w, int h) {
  bool out = false;
  for (int j = 0; j < 4; ++j) {
    const float x = (float)p[2 * j], y = (float)p[2 * j + 1];
    out |= x < kMinBorderDistance || x > (float)w - kMinBorderDistance || y < kMinBorderDistance || y > (float)h - kMinBorderDistance;
  }
  return out;
}

enum { kDropNone = 0, kDropBorder = 1, kDropNotGood = 2, kDropIdRange = 3 };
// the first rule that drops a decoded tag: 1. a corner within 4 px of the border, 2. not good, 3. id >= 36
ICC_HD int drop_reason(const double p[8], int hamming, int id, int w, int h) {
  if (near_border(p, w, h)) return kDropBorder;
  if (hamming > kErrorRecoveryBits) return kDropNotGood;
  if (id >= kIdLimit) return kDropIdRange;
  return kDropNone;
}

enum { kFrameFound = 0, kFrameFewTags = 1, kFrameDuplicate = 2 };
// 4. fewer than kMinTags tags left: nothing; 5. an id twice ("wild AprilTag"): nothing
ICC_HD int frame_verdict(int n_kept, const int* kept_ids) {
  if (n_kept < kMinTags) return kFrameFewTags;
  for (int i = 0; i < n_kept; ++i)
    for (int j = i + 1; j < n_kept; ++j)
      if (kept_ids[i] == kept_ids[j]) return kFrameDuplicate;
  return kFrameFound;
}

// ---- sub-pixel refinement: cv::cornerSubPix in FP64 ---------------------------------------------------------------------------
// The wrapper's window: r = max(2, 0.075 perimeter / 4 - 1) is the displacement limit, half-size ceil(r + 1), zero zone (-1, -1).
ICC_HD double subpix_radius(double perimeter) { return fmax(2.0, 7.5 / 100.0 * (perimeter / 4.0) - 1.0); }
ICC_HD int subpix_half_window(double radius) { return (int)ceil(radius + 1.0); }

// the image at (x, y), bilinear with the border replicated (cv::getRectSubPix)
ICC_HD double sample_replicate(const uint8_t* img, int64_t pitch, int w, int h, double x, double y) {
  const double fx = floor(x), fy = floor(y);
  const double ax = x - fx, ay = y - fy;
  const int x0 = (int)fx, y0 = (int)fy;
  const int xa = min(max(x0, 0), w - 1), xb = min(max(x0 + 1, 0), w - 1), ya = min(max(y0, 0), h - 1), yb = min(max(y0 + 1, 0), h - 1);
  const uint8_t* r0 = img + (int64_t)ya * pitch;
  const uint8_t* r1 = img + (int64_t)yb * pitch;
  return (1 - ay) * ((1 - ax) * r0[xa] + ax * r0[xb]) + ay * ((1 - ax) * r1[xa] + ax * r1[xb]);
}

// s += cornerSubPix's sums over window pixels k = first, first + stride, ... of (2 win + 1)^2 around c: s = {a, b, c, bb1, bb2}.
// Gradients are differences of bilinear samples one pixel either side; the weight is exp(-(px / win)^2 - (py / win)^2).
ICC_HD void subpix_accumulate(const uint8_t* img, int64_t pitch, int w, int h, double cx, double cy, int win, int first, int stride, double s[5]) {
  const int side = 2 * win + 1;
  for (int k = first; k < side * side; k += stride) {
    const int px = k % side - win, py = k / side - win;
    const double x = cx + px, y = cy + py;
    const double gx = sample_replicate(img, pitch, w, h, x + 1, y) - sample_replicate(img, pitch, w, h, x - 1, y);
    const double gy = sample_replicate(img, pitch, w, h, x, y + 1) - sample_replicate(img, pitch, w, h, x, y - 1);
    const double ux = (double)px / win, uy = (double)py / win;
    const double m = exp(-uy * uy) * exp(-ux * ux);
    const double gxx = gx * gx * m, gxy = gx * gy * m, gyy = gy * gy * m;
    s[0] += gxx; s[1] += gxy; s[2] += gyy;
    s[3] += gxx * px + gxy * py; s[4] += gxy * px + gyy * py;
  }
}

// one cornerSubPix update of the estimate (kept in float, as cv::Point2f); false when the system is singular (the loop stops)
ICC_HD bool subpix_update(const double s[5], float& cx, float& cy, double& err) {
  const double det = s[0] * s[2] - s[1] * s[1];
  if (fabs(det) <= 2.220446049250313e-16 * 2.220446049250313e-16) return false;
  const double scale = 1.0 / det;
  const float nx = (float)(cx + s[2] * scale * s[3] - s[1] * scale * s[4]);
  const float ny = (float)(cy - s[1] * scale * s[3] + s[0] * scale * s[4]);
  err = ((double)nx - cx) * ((double)nx - cx) + ((double)ny - cy) * ((double)ny - cy);
  cx = nx; cy = ny;
  return true;
}

// after the loop: an estimate that left the window falls back to the start
ICC_HD void subpix_finish(float sx, float sy, int win, float& cx, float& cy) {
  if (fabs((double)cx - sx) > win || fabs((double)cy - sy) > win) { cx = sx; cy = sy; }
}

}  // namespace aprilgrid
}  // namespace icc
