// Host-side test shim for the product's AprilGrid math (csrc/icc_aprilgrid_math.cuh): the functions the kernels of icc_aprilgrid.cu
// inline, compiled for the CPU by nvcc so that the `-m "not gpu"` suite can check them against OpenCV and NumPy.
#include "../../openimucameracalibrator_b200/csrc/icc_aprilgrid_math.cuh"

using namespace icc;
using namespace icc::aprilgrid;

static const uint64_t kCodes[kTag36h11Count] = {ICC_TAG36H11_CODES};

extern "C" {
int ag_code_count() { return kTag36h11Count; }
uint64_t ag_code(int i) { return kCodes[i]; }
uint64_t ag_rotate90(uint64_t w) { return rotate90(w); }
// decode_kernel for one quad q (x, y) x 4 in the quad frame's order: out = {id, hamming, rot, read code ok}; code_out the bits read
void ag_decode(const uint8_t* img, int w, int h, const double* q, int* out, uint64_t* code_out) {
  const QuadMap M = quad_map(q);
  double sb[kGraySums] = {0}, sw[kGraySums] = {0};
  for (int k = 0; k < kModelSamples; ++k) {
    int ix, iy;
    const int kind = model_kind(k, ix, iy);
    if (!kind) continue;
    const double x = (ix + 0.5) / kCells, y = (iy + 0.5) / kCells;
    double v;
    if (sample_pixel(img, w, w, h, M, x, y, v)) gray_add(kind == 2 ? sw : sb, x, y, v);
  }
  double cb[4], cw[4];
  gray_solve(sb, cb); gray_solve(sw, cw);
  uint64_t code = 0; int ok = 1;
  for (int k = 0; k < kDim * kDim; ++k) {
    double x, y, v;
    bit_position(k, x, y);
    const bool in = sample_pixel(img, w, w, h, M, x, y, v);
    ok &= in;
    code = (code << 1) | (uint64_t)(in && v > 0.5 * (gray_eval(cb, x, y) + gray_eval(cw, x, y)));
  }
  int ham, id, rot;
  unpack_key(decode_key(code, kCodes, 0, 1), ham, id, rot);
  out[0] = id; out[1] = ham; out[2] = rot; out[3] = ok;
  *code_out = code;
}
// refine_kernel for one corner from (x0, y0) with window half-size win: out = the refined corner; returns the iterations
int ag_corner_subpix(const uint8_t* img, int w, int h, float x0, float y0, int win, float* out) {
  float cx = x0, cy = y0;
  int it = 0;
  for (; it < kSubpixMaxIters;) {
    double s[5] = {0, 0, 0, 0, 0};
    subpix_accumulate(img, w, w, h, cx, cy, win, 0, 1, s);
    double err;
    if (!subpix_update(s, cx, cy, err)) break;
    ++it;
    if (cx < 0 || cx >= w || cy < 0 || cy >= h) break;
    if (err <= kSubpixEps * kSubpixEps) break;
  }
  subpix_finish(x0, y0, win, cx, cy);
  out[0] = cx; out[1] = cy;
  return it;
}
double ag_subpix_radius(double perimeter) { return subpix_radius(perimeter); }
int ag_subpix_half_window(double r) { return subpix_half_window(r); }
int ag_drop_reason(const double* p, int hamming, int id, int w, int h) { return drop_reason(p, hamming, id, w, h); }
int ag_frame_verdict(int n, const int* ids) { return frame_verdict(n, ids); }
}
