// Host-side test shim for the colour stage of the radon-board extraction (icc_board_math.cuh: bgr_resize_gray_pixel), compiled for the
// CPU by nvcc so that the `-m "not gpu"` suite can compare it with committed cv2 output.
#include "../../openimucameracalibrator_b200/csrc/icc_board_math.cuh"

using namespace icc;

extern "C" {
// cvtColor(resize(bgr, 1/f), BGR2GRAY) as bgr_gray_kernel computes it: bgr is h rows of `pitch` bytes, dst resize_dim(h) x resize_dim(w)
void bm_bgr_resize_gray(const uint8_t* bgr, int64_t pitch, int w, int h, double f, uint8_t* dst) {
  const int dw = f == 1.0 ? w : board::resize_dim(w, f), dh = f == 1.0 ? h : board::resize_dim(h, f);
  for (int y = 0; y < dh; ++y)
    for (int x = 0; x < dw; ++x) dst[(int64_t)y * dw + x] = board::bgr_resize_gray_pixel(bgr, pitch, w, h, f, x, y);
}
}
