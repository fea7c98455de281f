// Per-pixel and per-corner math of the radon checkerboard extraction (icc_board.cu), kept in a header so that
// tests/board/board_host_math.cu compiles exactly this code for the CPU.
//
// Reference: BoardExtractor::ExtractBoard with BoardType::RADON (src/core/board_extractor.cc), i.e. cv::resize and
// cv::findChessboardCornersSB(CALIB_CB_LARGER | CALIB_CB_MARKER | CALIB_CB_EXHAUSTIVE).
#pragma once
#include "icc_device_math.cuh"

#include <cmath>
#include <cstdint>

namespace icc {
namespace board {

// ---- downsampling: cv::resize(img, img, Size(), 1/f, 1/f) with INTER_LINEAR on 8-bit gray --------------------------------------
// OpenCV takes dst = cvRound(src / f) (ties to even) and scale = 1 / (1 / f).  Exactly scale 2 becomes INTER_AREA's fast 2x2 mean
// (S00 + S01 + S10 + S11 + 2) >> 2; any other scale is the fixed-point bilinear filter: source coordinate (d + 0.5) scale - 0.5 in
// float, 11-bit weights rounded to even, the horizontal sum in int, and the vertical pass ((b0 (S0 >> 4)) >> 16) +
// ((b1 (S1 >> 4)) >> 16) + 2) >> 2.  Columns past the last source pixel take it with weight 2048; rows clamp to the image.
ICC_HD int resize_dim(int src, double f) { return (int)nearbyint((double)src * (1.0 / f)); }
ICC_HD double resize_scale(double f) { return 1.0 / (1.0 / f); }
ICC_HD bool resize_is_area2(double f) { return resize_scale(f) == 2.0; }

// source index and 11-bit weight of output coordinate d (the clamp of the column coefficients; rows are clamped by the caller)
ICC_HD void resize_coeff(int d, double scale, int ssize, bool clamp_hi, int& s, int& w0, int& w1) {
  float fx = (float)((d + 0.5) * scale - 0.5);
  s = (int)floorf(fx);
  fx -= (float)s;
  if (s < 0) { fx = 0.f; s = 0; }
  if (clamp_hi && s >= ssize - 1) { fx = 0.f; s = ssize - 1; }
  w0 = (int)rintf((1.f - fx) * 2048.f);
  w1 = (int)rintf(fx * 2048.f);
}

// one channel of pixels STEP bytes apart (1: gray; 3: one channel of interleaved B, G, R, src pointing at that channel's first byte)
template <int STEP>
ICC_HD uint8_t resize_channel(const uint8_t* src, int64_t pitch, int sw, int sh, double f, int dx, int dy) {
  const double scale = resize_scale(f);
  if (scale == 2.0) {
    const int sx = 2 * dx, sy = 2 * dy;
    if (sx + 1 < sw && sy + 1 < sh) {
      const uint8_t* r0 = src + (int64_t)sy * pitch + (int64_t)sx * STEP;
      return (uint8_t)((r0[0] + r0[STEP] + r0[pitch] + r0[pitch + STEP] + 2) >> 2);
    }
    int sum = 0, cnt = 0;   // resizeAreaFast_'s border: the mean of the block's pixels inside the image
    for (int y = sy; y < sy + 2 && y < sh; ++y)
      for (int x = sx; x < sx + 2 && x < sw; ++x) { sum += src[(int64_t)y * pitch + (int64_t)x * STEP]; ++cnt; }
    return (uint8_t)min(255, max(0, (int)rintf((float)sum / (float)cnt)));
  }
  int sx, a0, a1, sy, b0, b1;
  resize_coeff(dx, scale, sw, true, sx, a0, a1);
  resize_coeff(dy, scale, sh, false, sy, b0, b1);
  const int sx1 = min(sx + 1, sw - 1), y0 = min(max(sy, 0), sh - 1), y1 = min(max(sy + 1, 0), sh - 1);
  const uint8_t* r0 = src + (int64_t)y0 * pitch;
  const uint8_t* r1 = src + (int64_t)y1 * pitch;
  const int S0 = r0[sx * STEP] * a0 + r0[sx1 * STEP] * a1, S1 = r1[sx * STEP] * a0 + r1[sx1 * STEP] * a1;
  return (uint8_t)((((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2);
}

ICC_HD uint8_t resize_pixel(const uint8_t* src, int64_t pitch, int sw, int sh, double f, int dx, int dy) {
  return resize_channel<1>(src, pitch, sw, sh, f, dx, dy);
}

// ---- colour frames: cv::resize on the BGR image, then cv::cvtColor(BGR2GRAY) ----------------------------------------------------
// The reference resizes the colour image and converts afterwards (BoardExtractor::ExtractImageFolderToJson), which is not the same
// image as converting first.  OpenCV's 8UC3 resize is three independent single-channel resizes.  OpenCV 4.13's 8-bit BGR2GRAY is the
// 15-bit fixed-point rule (B 3735 + G 19235 + R 9798 + 2^14) >> 15 (with or without IPP); the often-quoted 14-bit weights
// 1868 / 9617 / 4899 differ on about 0.26 % of pixels.  B = G = R = v gives v exactly, so a gray image converts to itself.
ICC_HD uint8_t bgr_to_gray(int b, int g, int r) { return (uint8_t)((b * 3735 + g * 19235 + r * 9798 + 16384) >> 15); }

// output pixel (dx, dy) of cvtColor(resize(bgr, 1/f), BGR2GRAY); pitch in bytes (>= 3 sw); at f = 1 only the conversion
ICC_HD uint8_t bgr_resize_gray_pixel(const uint8_t* bgr, int64_t pitch, int sw, int sh, double f, int dx, int dy) {
  if (f == 1.0) { const uint8_t* p = bgr + (int64_t)dy * pitch + 3 * (int64_t)dx; return bgr_to_gray(p[0], p[1], p[2]); }
  return bgr_to_gray(resize_channel<3>(bgr, pitch, sw, sh, f, dx, dy), resize_channel<3>(bgr + 1, pitch, sw, sh, f, dx, dy),
                     resize_channel<3>(bgr + 2, pitch, sw, sh, f, dx, dy));
}

// ---- corner response: a localized Radon transform on a 3x3 box mean (Duda & Frese, BMVC 2018) -------------------------------------
// B = the 3x3 box mean of the image.  L_k(p) = sum over t = -R..R of B(p + t d_k) along d_k = (1, 0), (1, 1), (0, 1), (-1, 1); the
// response is (max_k L_k - min_k L_k)^2 / (2R + 1)^2.  At an X-junction one diagonal line runs through the two dark squares and the
// other through the two light ones; along an edge or in a flat region the four sums agree.  Pixels closer than R + 1 to the border
// have response 0.
constexpr int kRadonR = 4;
constexpr int kBorder = kRadonR + 1;

ICC_HD float box3(const uint8_t* img, int64_t pitch, int x, int y) {
  int s = 0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) s += img[(int64_t)(y + dy) * pitch + x + dx];
  return (float)s * (1.f / 9.f);
}

// box: the 3x3 box mean (pitch in floats); valid for kBorder <= x < w - kBorder, likewise y
ICC_HD float radon_response(const float* box, int64_t pitch, int x, int y) {
  const int ddx[4] = {1, 1, 0, -1}, ddy[4] = {0, 1, 1, 1};
  float lo = 3.4e38f, hi = -3.4e38f;
  for (int k = 0; k < 4; ++k) {
    float s = 0.f;
    for (int t = -kRadonR; t <= kRadonR; ++t) s += box[(int64_t)(y + t * ddy[k]) * pitch + x + t * ddx[k]];
    lo = fminf(lo, s); hi = fmaxf(hi, s);
  }
  const float d = (hi - lo) * (1.f / (2 * kRadonR + 1));
  return d * d;
}

// ---- sub-pixel refinement: gradient orthogonality (Foerstner; cv::cornerSubPix without a zero zone) --------------------------------
// The window is the pixels p = (round(qx) + dx, round(qy) + dy), |dx|, |dy| <= hw + hw / 2 (3 sigma), around the estimate q.  Each contributes its
// central-difference gradient g (at the pixel itself: no interpolation, which would bias the estimate by the sub-pixel phase) with
// Gaussian weight exp(-|p - q|^2 / (2 (hw / 2)^2)); the new estimate solves (sum w g g^T) q' = sum w g g^T p in FP64.  Iterated until
// the step is below kSubpixEps or kSubpixIters steps.  The window is clamped so that every gradient stays inside the image.
constexpr double kSubpixEps = 1e-3;
constexpr int kSubpixIters = 40;

ICC_HD double sample_bilinear(const uint8_t* img, int64_t pitch, int w, int h, double x, double y) {
  x = fmin(fmax(x, 0.0), w - 1.0); y = fmin(fmax(y, 0.0), h - 1.0);
  const int x0 = min((int)x, w - 2), y0 = min((int)y, h - 2);
  const double ax = x - x0, ay = y - y0;
  const uint8_t* r0 = img + (int64_t)y0 * pitch + x0;
  const uint8_t* r1 = r0 + pitch;
  return (1 - ay) * ((1 - ax) * r0[0] + ax * r0[1]) + ay * ((1 - ax) * r1[0] + ax * r1[1]);
}

// s += the window pixels k = first, first + stride, ... (of (2 (hw + hw / 2) + 1)^2) around q: s = {a11, a12, a22, b1, b2}
ICC_HD void subpix_accumulate(const uint8_t* img, int64_t pitch, int w, int h, double qx, double qy, int hw, int first, int stride, double s[5]) {
  const int half = hw + hw / 2, side = 2 * half + 1;
  const double inv2s2 = 2.0 / ((double)hw * hw);   // 1 / (2 sigma^2), sigma = hw / 2
  const int cx = (int)floor(qx + 0.5), cy = (int)floor(qy + 0.5);
  for (int k = first; k < side * side; k += stride) {
    const int px = cx + k % side - half, py = cy + k / side - half;
    if (px < 1 || py < 1 || px > w - 2 || py > h - 2) continue;
    const uint8_t* r = img + (int64_t)py * pitch + px;
    const double gx = 0.5 * ((double)r[1] - (double)r[-1]);
    const double gy = 0.5 * ((double)r[pitch] - (double)r[-pitch]);
    const double ex = px - qx, ey = py - qy;
    const double wt = exp(-(ex * ex + ey * ey) * inv2s2);
    const double gxx = wt * gx * gx, gxy = wt * gx * gy, gyy = wt * gy * gy;
    s[0] += gxx; s[1] += gxy; s[2] += gyy;
    s[3] += gxx * px + gxy * py; s[4] += gxy * px + gyy * py;
  }
}

// the 2x2 solve of the accumulated sums; false when the system is singular
ICC_HD bool subpix_solve(const double s[5], double& qx, double& qy) {
  const double det = s[0] * s[2] - s[1] * s[1];
  if (!(fabs(det) > 1e-12 * (s[0] * s[2] + 1e-300))) return false;
  qx = (s[2] * s[3] - s[1] * s[4]) / det;
  qy = (s[0] * s[4] - s[1] * s[3]) / det;
  return true;
}

// window half-size for a corner whose nearest grid neighbour is `spacing` px away: 0.35 squares keeps the neighbouring corners
// and the marker circles out of the window
ICC_HD int subpix_half_window(float spacing) { return max(2, min(12, (int)(0.35f * spacing))); }

}  // namespace board
}  // namespace icc
