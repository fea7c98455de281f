// Host-side test shim for the product's radon-board math (csrc/icc_board_math.cuh): the functions the kernels of icc_board.cu
// inline, compiled for the CPU by nvcc so that the `-m "not gpu"` suite can compare them with NumPy statements of the same rules.
#include "../../openimucameracalibrator_b200/csrc/icc_board_math.cuh"

using namespace icc;

extern "C" {
// cv::resize(src, 1/f) as resize_kernel computes it; dst is resize_dim(h) x resize_dim(w), packed
void bm_resize(const uint8_t* src, int64_t pitch, int w, int h, double f, uint8_t* dst) {
  const int dw = board::resize_dim(w, f), dh = board::resize_dim(h, f);
  for (int y = 0; y < dh; ++y)
    for (int x = 0; x < dw; ++x) dst[(int64_t)y * dw + x] = board::resize_pixel(src, pitch, w, h, f, x, y);
}
int bm_resize_dim(int n, double f) { return board::resize_dim(n, f); }
// box_kernel + response_kernel: the response image (w x h floats, 0 on the border)
void bm_response(const uint8_t* img, int w, int h, float* box, float* resp) {
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) box[(int64_t)y * w + x] = (x >= 1 && y >= 1 && x < w - 1 && y < h - 1) ? board::box3(img, w, x, y) : 0.f;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const bool in = x >= board::kBorder && y >= board::kBorder && x < w - board::kBorder && y < h - board::kBorder;
      resp[(int64_t)y * w + x] = in ? board::radon_response(box, w, x, y) : 0.f;
    }
}
// refine_kernel for one corner: the iterations until the step is below kSubpixEps; returns the iterations taken
int bm_refine(const uint8_t* img, int w, int h, double x0, double y0, float spacing, double* out) {
  const int hw = board::subpix_half_window(spacing);
  double qx = x0, qy = y0;
  int it = 0;
  for (; it < board::kSubpixIters; ++it) {
    double s[5] = {0, 0, 0, 0, 0};
    board::subpix_accumulate(img, w, w, h, qx, qy, hw, 0, 1, s);
    double nx, ny;
    if (!board::subpix_solve(s, nx, ny)) break;
    const double step = hypot(nx - qx, ny - qy);
    if (step > hw) break;
    qx = nx; qy = ny;
    if (step < board::kSubpixEps) { ++it; break; }
  }
  out[0] = qx; out[1] = qy;
  return it;
}
// one accumulate + solve at q; returns 0 when the system is singular
int bm_subpix_step(const uint8_t* img, int w, int h, double qx, double qy, int hw, double* out) {
  double s[5] = {0, 0, 0, 0, 0};
  board::subpix_accumulate(img, w, w, h, qx, qy, hw, 0, 1, s);
  return board::subpix_solve(s, out[0], out[1]) ? 1 : 0;
}
int bm_half_window(float spacing) { return board::subpix_half_window(spacing); }
}
