// Radon checkerboard corner extraction on the GPU (sm_90a): what the reference's extract_board_to_json computes per frame with
// --board_type radon, i.e. BoardExtractor::ExtractBoard -> cv::findChessboardCornersSB(CALIB_CB_LARGER | CALIB_CB_MARKER |
// CALIB_CB_EXHAUSTIVE) on the optionally cv::resize'd frame (src/core/board_extractor.cc).
//
// Frames go through in chunks of kChunk (ICC_BOARD_CHUNK_FRAMES overrides it), so device memory stays bounded whatever the count.
// Per chunk:
//   resize_kernel     cv::resize INTER_LINEAR (icc_board_math.cuh), skipped at f = 1; for colour frames bgr_gray_kernel instead:
//                     cv::resize of each B, G, R channel, then OpenCV's BGR2GRAY (at f = 1 only the conversion);
//   box_kernel        the 3x3 box mean, FP32;
//   response_kernel   the localized Radon response, and the frame's maximum (atomicMax on the float's bits: responses are >= 0);
//   candidate_kernel  one CTA per 32x32 tile: a pixel is a candidate when its response is >= kRelThreshold x the frame maximum and
//                     the largest in its 7x7 neighbourhood (ties to the lower pixel index); candidates are appended to the frame's
//                     list of kMaxCandidates, and the ones past it are counted;
//   grid_kernel       one warp per frame: grows a grid from a seed, checks the W x H count and the three markers, and orders the
//                     corners by the markers (below);
//   refine_kernel     one warp per corner of a found frame: gradient-orthogonality refinement in FP64.
// Every choice among candidates breaks ties on the pixel index, so the result does not depend on the order of the list, on the
// chunking or on where the frames came from.
#include "../../include/icc_b200.h"
#include "icc_board_math.cuh"
#include "icc_host.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

namespace icc {

namespace {

constexpr int kChunk = 32;
constexpr int kMaxCandidates = 1024;
constexpr float kRelThreshold = 0.4f;
constexpr int kNms = 3;                  // 7x7 neighbourhood
constexpr int kTile = 32;
constexpr int kMaxSide = 32;             // grid coordinates stay in (-kMaxSide, kMaxSide)
constexpr int kGridDim = 2 * kMaxSide - 1;
constexpr float kSearch = 0.35f;         // a predicted corner takes the nearest candidate within kSearch x the local step
enum { kFound = 0, kNoGrid = 1, kWrongCount = 2, kNoMarkers = 3 };

struct Cand { float x, y, r; int key; };   // key = y * width + x

__global__ void resize_kernel(const uint8_t* __restrict__ src, int sw, int sh, double f, uint8_t* __restrict__ dst, int dw, int dh) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= dw || y >= dh) return;
  dst[((size_t)n * dh + y) * dw + x] = board::resize_pixel(src + (size_t)n * sw * sh, sw, sw, sh, f, x, y);
}

__global__ void bgr_gray_kernel(const uint8_t* __restrict__ src, int sw, int sh, double f, uint8_t* __restrict__ dst, int dw, int dh) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= dw || y >= dh) return;
  dst[((size_t)n * dh + y) * dw + x] = board::bgr_resize_gray_pixel(src + (size_t)n * 3 * sw * sh, 3 * (int64_t)sw, sw, sh, f, x, y);
}

__global__ void box_kernel(const uint8_t* __restrict__ img, int w, int h, float* __restrict__ box) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= w || y >= h) return;
  const bool in = x >= 1 && y >= 1 && x < w - 1 && y < h - 1;
  box[((size_t)n * h + y) * w + x] = in ? board::box3(img + (size_t)n * w * h, w, x, y) : 0.f;
}

__global__ void response_kernel(const float* __restrict__ box, int w, int h, float* __restrict__ resp, unsigned* __restrict__ fmax) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  float r = 0.f;
  if (x >= board::kBorder && y >= board::kBorder && x < w - board::kBorder && y < h - board::kBorder) r = board::radon_response(box + (size_t)n * w * h, w, x, y);
  if (x < w && y < h) resp[((size_t)n * h + y) * w + x] = r;
  for (int o = 16; o; o >>= 1) r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
  if ((threadIdx.x & 31) == 0 && r > 0.f) atomicMax(fmax + n, __float_as_uint(r));
}

__global__ void __launch_bounds__(256) candidate_kernel(const float* __restrict__ resp, int w, int h, const unsigned* __restrict__ fmax, Cand* __restrict__ cand,
                                                        int* __restrict__ count, int* __restrict__ overflow) {
  __shared__ float t[kTile + 2 * kNms][kTile + 2 * kNms];
  const int n = blockIdx.z, x0 = blockIdx.x * kTile - kNms, y0 = blockIdx.y * kTile - kNms;
  const float* R = resp + (size_t)n * w * h;
  for (int i = threadIdx.x; i < (kTile + 2 * kNms) * (kTile + 2 * kNms); i += blockDim.x) {
    const int tx = i % (kTile + 2 * kNms), ty = i / (kTile + 2 * kNms), x = x0 + tx, y = y0 + ty;
    t[ty][tx] = (x >= 0 && y >= 0 && x < w && y < h) ? R[(size_t)y * w + x] : 0.f;
  }
  __syncthreads();
  const float thr = kRelThreshold * __uint_as_float(fmax[n]);
  for (int i = threadIdx.x; i < kTile * kTile; i += blockDim.x) {
    const int tx = i % kTile + kNms, ty = i / kTile + kNms, x = x0 + tx, y = y0 + ty;
    if (x >= w || y >= h) continue;
    const float v = t[ty][tx];
    if (!(v > 0.f) || v < thr) continue;
    bool peak = true;
    for (int dy = -kNms; dy <= kNms && peak; ++dy)
      for (int dx = -kNms; dx <= kNms; ++dx) {
        const float u = t[ty + dy][tx + dx];
        if (u > v || (u == v && (dy < 0 || (dy == 0 && dx < 0)))) { peak = false; break; }
      }
    if (!peak) continue;
    const int slot = atomicAdd(count + n, 1);
    if (slot < kMaxCandidates) cand[(size_t)n * kMaxCandidates + slot] = Cand{(float)x, (float)y, v, y * w + x};
    else atomicAdd(overflow + n, 1);
  }
}

// (a, key) < (b, bkey) lexicographically; the warp's minimum of (a, key) over its lanes
ICC_D void warp_argmin(float& a, int& key, int& idx) {
  for (int o = 16; o; o >>= 1) {
    const float a2 = __shfl_xor_sync(0xffffffffu, a, o);
    const int k2 = __shfl_xor_sync(0xffffffffu, key, o), i2 = __shfl_xor_sync(0xffffffffu, idx, o);
    if (a2 < a || (a2 == a && k2 < key)) { a = a2; key = k2; idx = i2; }
  }
}

struct GridArgs {
  const Cand* cand; const int* count; const uint8_t* img; int w, h, W, H;
  float2* corner;          // per frame W*H integer-pixel corners in id order
  float* spacing;          // per corner: distance to its nearest grid neighbour
  int* status;             // per frame kFound / kNoGrid / kWrongCount / kNoMarkers
};

// One warp per frame.  The seed is the strongest candidate (ties to the lower pixel index); its nearest candidate fixes the first
// grid axis and the nearest one at more than 60 degrees from it the second.  The grid then grows breadth-first: the corner next to a
// placed corner P along an axis is predicted as 2P - (P's predecessor on that axis) when there is one, as P plus the step of the
// parallel row or column next to it otherwise, and takes the nearest unused candidate within kSearch x that step.  Predicting from
// the neighbours only, never from one homography, follows the lines of a fisheye image.  The frame is found iff the placed
// corners fill a W x H (or H x W) box exactly and the three markers are found where the board has them.
__global__ void __launch_bounds__(32) grid_kernel(GridArgs A) {
  __shared__ Cand c[kMaxCandidates];
  __shared__ short cell[kGridDim * kGridDim];       // candidate index + 1 at grid position, 0 when empty
  __shared__ short queue[kMaxCandidates];
  __shared__ unsigned char used[kMaxCandidates];
  __shared__ float S[kMaxSide * kMaxSide], Cc[kMaxSide * kMaxSide];
  const int n = blockIdx.x, lane = threadIdx.x;
  const int nc = min(A.count[n], kMaxCandidates);
  for (int i = lane; i < nc; i += 32) { c[i] = A.cand[(size_t)n * kMaxCandidates + i]; used[i] = 0; }
  for (int i = lane; i < kGridDim * kGridDim; i += 32) cell[i] = 0;
  __syncwarp();
  const int W = A.W, H = A.H;
  if (lane == 0) A.status[n] = kNoGrid;
  if (nc < W * H) return;
  // seed: strongest candidate
  float best = 0.f; int bkey = 0x7fffffff, bi = -1;
  for (int i = lane; i < nc; i += 32) { const float v = -c[i].r; if (bi < 0 || v < best || (v == best && c[i].key < bkey)) { best = v; bkey = c[i].key; bi = i; } }
  warp_argmin(best, bkey, bi);
  const int seed = bi;
  auto nearest = [&](float px, float py, float maxd2, float dirx, float diry, float maxcos2) {
    float bd = 3.4e38f; int k = 0x7fffffff, idx = -1;
    for (int i = lane; i < nc; i += 32) {
      if (used[i]) continue;
      const float dx = c[i].x - px, dy = c[i].y - py, d2 = dx * dx + dy * dy;
      if (d2 > maxd2) continue;
      if (maxcos2 < 1.f) { const float dt = dx * dirx + dy * diry; if (dt * dt > maxcos2 * d2 * (dirx * dirx + diry * diry)) continue; }
      if (d2 < bd || (d2 == bd && c[i].key < k)) { bd = d2; k = c[i].key; idx = i; }
    }
    warp_argmin(bd, k, idx);
    return idx;
  };
  const float sx = c[seed].x, sy = c[seed].y;
  if (lane == 0) used[seed] = 1;
  __syncwarp();
  const int n1 = nearest(sx, sy, 3.4e38f, 0.f, 0.f, 1.f);
  if (n1 < 0) return;
  const float ax = c[n1].x - sx, ay = c[n1].y - sy;
  const int n2 = nearest(sx, sy, 4.f * (ax * ax + ay * ay), ax, ay, 0.25f);
  if (n2 < 0) return;
  const int o = kMaxSide - 1;
  auto at = [&](int u, int v) -> int { return (u <= -kMaxSide || v <= -kMaxSide || u >= kMaxSide || v >= kMaxSide) ? -2 : (int)cell[(v + o) * kGridDim + u + o] - 1; };
  auto cu = [&](int q) { return (int)(q % kGridDim) - o; };
  auto cv = [&](int q) { return (int)(q / kGridDim) - o; };
  int qn = 0;
  if (lane == 0) {
    cell[o * kGridDim + o] = seed + 1; cell[o * kGridDim + o + 1] = n1 + 1; cell[(o + 1) * kGridDim + o] = n2 + 1;
    used[n1] = used[n2] = 1;
    queue[0] = o * kGridDim + o; queue[1] = o * kGridDim + o + 1; queue[2] = (o + 1) * kGridDim + o;
  }
  qn = 3;
  __syncwarp();
  int umin = 0, umax = 1, vmin = 0, vmax = 1;
  for (int qh = 0; qh < qn; ++qh) {
    const int q = queue[qh], u = cu(q), v = cv(q);
    const int pi = at(u, v);
    for (int d = 0; d < 4; ++d) {
      const int eu = d == 0 ? 1 : d == 1 ? -1 : 0, ev = d == 2 ? 1 : d == 3 ? -1 : 0;
      const int tu = u + eu, tv = v + ev;
      if (at(tu, tv) != -1) continue;   // occupied or outside the table
      if (max(umax, tu) - min(umin, tu) >= max(W, H) || max(vmax, tv) - min(vmin, tv) >= max(W, H)) continue;
      float stx, sty; bool have = false;
      const int back = at(u - eu, v - ev);
      if (back >= 0) { stx = c[pi].x - c[back].x; sty = c[pi].y - c[back].y; have = true; }
      for (int side = -1; side <= 1 && !have; side += 2) {   // the parallel line next to P: its step from (u + side e_perp) to (t + side e_perp)
        const int a = at(u + side * ev, v + side * eu), b = at(tu + side * ev, tv + side * eu);
        if (a >= 0 && b >= 0) { stx = c[b].x - c[a].x; sty = c[b].y - c[a].y; have = true; }
      }
      if (!have) {   // the seed's axes
        if (eu) { stx = eu * ax; sty = eu * ay; } else { stx = ev * (c[n2].x - sx); sty = ev * (c[n2].y - sy); }
      }
      const float px = c[pi].x + stx, py = c[pi].y + sty, r2 = kSearch * kSearch * (stx * stx + sty * sty);
      const int k = nearest(px, py, r2, 0.f, 0.f, 1.f);
      if (k < 0) continue;
      if (lane == 0) { cell[(tv + o) * kGridDim + tu + o] = k + 1; used[k] = 1; queue[qn] = (tv + o) * kGridDim + tu + o; }
      __syncwarp();
      ++qn;
      umin = min(umin, tu); umax = max(umax, tu); vmin = min(vmin, tv); vmax = max(vmax, tv);
      if (qn >= kMaxCandidates) break;
    }
    if (qn >= kMaxCandidates) break;
  }
  const int bw = umax - umin + 1, bh = vmax - vmin + 1;
  if (lane == 0) A.status[n] = qn < 9 ? kNoGrid : kWrongCount;
  if (!(qn == W * H && ((bw == W && bh == H) || (bw == H && bh == W)))) return;
  // ---- markers: per cell, the mean of four samples 0.55 of the way to the corners (the square) and the centre sample ----------
  const int ncu = bw - 1, ncv = bh - 1, ncell = ncu * ncv;
  auto P = [&](int u, int v) { const Cand& q = c[at(u + umin, v + vmin)]; return make_float2(q.x, q.y); };
  auto centre = [&](int cu_, int cv_) {
    const float2 a = P(cu_, cv_), b = P(cu_ + 1, cv_), d = P(cu_, cv_ + 1), e = P(cu_ + 1, cv_ + 1);
    return make_float2(0.25f * (a.x + b.x + d.x + e.x), 0.25f * (a.y + b.y + d.y + e.y));
  };
  const uint8_t* img = A.img + (size_t)n * A.w * A.h;
  float sum = 0.f;
  for (int k = lane; k < ncell; k += 32) {
    const int cu_ = k % ncu, cv_ = k / ncu;
    const float2 m = centre(cu_, cv_);
    float s = 0.f;
    for (int j = 0; j < 4; ++j) {
      const float2 p = P(cu_ + (j & 1), cv_ + (j >> 1));
      s += (float)board::sample_bilinear(img, A.w, A.w, A.h, m.x + 0.55f * (p.x - m.x), m.y + 0.55f * (p.y - m.y));
    }
    S[k] = 0.25f * s;
    Cc[k] = (float)board::sample_bilinear(img, A.w, A.w, A.h, m.x, m.y);
    sum += S[k];
  }
  for (int o2 = 16; o2; o2 >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o2);
  __syncwarp();
  const float T = sum / ncell;
  int nmark = 0, vtx = -1, arm0 = -1, arm1 = -1;   // warp-uniform after the loop (every lane walks all cells)
  for (int k = 0; k < ncell; ++k) {
    const bool dark = S[k] < T, mk = dark ? Cc[k] > T : Cc[k] < T;
    if (!mk) continue;
    ++nmark;
    if (!dark) vtx = k; else if (arm0 < 0) arm0 = k; else arm1 = k;
  }
  if (lane == 0) A.status[n] = kNoMarkers;
  if (nmark != 3 || vtx < 0 || arm1 < 0) return;
  const int vu = vtx % ncu, vv = vtx / ncu;
  const int a0u = arm0 % ncu - vu, a0v = arm0 / ncu - vv, a1u = arm1 % ncu - vu, a1v = arm1 / ncu - vv;
  if (abs(a0u) + abs(a0v) != 1 || abs(a1u) + abs(a1v) != 1 || a0u * a1u + a0v * a1v != 0) return;   // two perpendicular unit arms
  // the +i arm U and the +j arm R of the board satisfy cross(U - V, R - V) > 0 in the image (x right, y down)
  const float2 mv = centre(vu, vv), m0 = centre(vu + a0u, vv + a0v), m1 = centre(vu + a1u, vv + a1v);
  const float cr = (m0.x - mv.x) * (m1.y - mv.y) - (m0.y - mv.y) * (m1.x - mv.x);
  const int iu = cr > 0.f ? a0u : a1u, iv = cr > 0.f ? a0v : a1v, ju = cr > 0.f ? a1u : a0u, jv = cr > 0.f ? a1v : a0v;
  // board cell (H / 2 - 1, W / 2 - 1) is the vertex; its corner from which +i and +j stay in the cell is board corner (H / 2 - 1, W / 2 - 1)
  const int bi0 = H / 2 - 1, bj0 = W / 2 - 1;
  const int g0u = vu + ((iu + ju) > 0 ? 0 : 1) - bi0 * iu - bj0 * ju, g0v = vv + ((iv + jv) > 0 ? 0 : 1) - bi0 * iv - bj0 * jv;
  // the markers are in their squares iff every board corner lands in the grid: a mirrored board (seen from the back, or a flipped
  // camera) or an L in another cell maps some ids outside it
  const int e0u = g0u + (H - 1) * iu, e0v = g0v + (H - 1) * iv, e1u = g0u + (W - 1) * ju, e1v = g0v + (W - 1) * jv;
  const int e2u = e0u + (W - 1) * ju, e2v = e0v + (W - 1) * jv;
  auto inside = [&](int u, int v) { return u >= 0 && v >= 0 && u < bw && v < bh; };
  if (!inside(g0u, g0v) || !inside(e0u, e0v) || !inside(e1u, e1v) || !inside(e2u, e2v)) return;
  for (int id = lane; id < W * H; id += 32) {
    const int i = id / W, j = id % W, gu = g0u + i * iu + j * ju, gv = g0v + i * iv + j * jv;
    const float2 p = P(gu, gv);
    float sp = 3.4e38f;
    {
      for (int d = 0; d < 4; ++d) {
        const int nu = gu + (d == 0) - (d == 1), nv = gv + (d == 2) - (d == 3);
        if (nu < 0 || nv < 0 || nu >= bw || nv >= bh) continue;
        const float2 q = P(nu, nv); sp = fminf(sp, hypotf(q.x - p.x, q.y - p.y));
      }
    }
    A.corner[(size_t)n * W * H + id] = p; A.spacing[(size_t)n * W * H + id] = sp;
  }
  if (lane == 0) A.status[n] = kFound;
}

// one warp per corner of the chunk; corners of frames that were not found are skipped
__global__ void __launch_bounds__(128) refine_kernel(const uint8_t* __restrict__ img, int w, int h, int per_frame, int n_corners, const int* __restrict__ status,
                                                     const float2* __restrict__ corner, const float* __restrict__ spacing, double2* __restrict__ uv) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (g >= n_corners) return;
  const int n = g / per_frame;
  if (status[n] != kFound) return;
  const uint8_t* I = img + (size_t)n * w * h;
  const int hw = board::subpix_half_window(spacing[g]);
  double qx = corner[g].x, qy = corner[g].y;
  for (int it = 0; it < board::kSubpixIters; ++it) {
    double s[5] = {0, 0, 0, 0, 0};
    board::subpix_accumulate(I, w, w, h, qx, qy, hw, lane, 32, s);
    for (int k = 0; k < 5; ++k)
      for (int o = 16; o; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    double nx, ny;
    if (!board::subpix_solve(s, nx, ny)) break;
    const double step = hypot(nx - qx, ny - qy);
    if (step > hw) break;   // left the window: keep the last estimate
    qx = nx; qy = ny;
    if (step < board::kSubpixEps) break;
  }
  if (lane == 0) uv[g] = make_double2(qx, qy);
}

}  // namespace

#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status extract_radon_board(cudaStream_t st, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, bool frames_on_device, bool bgr, int W, int H,
                               double f, double* uv_out, int32_t* found, icc_board_summary& S, std::string& err) {
  const auto t0 = std::chrono::steady_clock::now();
  const int launches0 = kernel_launch_count();
  memset(&S, 0, sizeof S);
  const bool scaled = f != 1.0;
  const int w = scaled ? board::resize_dim(width, f) : width, h = scaled ? board::resize_dim(height, f) : height;
  S.width = w; S.height = h;
  if (w < 2 * board::kBorder + 2 || h < 2 * board::kBorder + 2) { err = "the (downsampled) frame is too small"; return ICC_ERR_INVALID_ARGUMENT; }
  if (W >= kMaxSide || H >= kMaxSide) { err = "corners_x and corners_y must be below 32"; return ICC_ERR_INVALID_ARGUMENT; }
  int chunk = kChunk;
  if (const char* e = getenv("ICC_BOARD_CHUNK_FRAMES")) chunk = std::max(1, atoi(e));
  chunk = std::min(chunk, std::max(n_frames, 1));
  const size_t row = (size_t)width * (bgr ? 3 : 1), in_bytes = row * height, px = (size_t)w * h, per = (size_t)W * H;
  DevBuf<uint8_t> d_in, d_small; DevBuf<float> d_box, d_resp, d_spacing; DevBuf<unsigned> d_max; DevBuf<Cand> d_cand;
  DevBuf<int> d_count, d_over, d_status; DevBuf<float2> d_corner; DevBuf<double2> d_uv;
  CU(d_in.alloc(chunk * in_bytes)); CU(d_box.alloc(chunk * px)); CU(d_resp.alloc(chunk * px)); CU(d_max.alloc(chunk));
  if (scaled || bgr) CU(d_small.alloc(chunk * px));
  CU(d_cand.alloc((size_t)chunk * kMaxCandidates)); CU(d_count.alloc(chunk)); CU(d_over.alloc(chunk)); CU(d_status.alloc(chunk));
  CU(d_corner.alloc(chunk * per)); CU(d_spacing.alloc(chunk * per)); CU(d_uv.alloc(chunk * per));
  std::vector<int> status(chunk), over(chunk);
  std::vector<double2> uv(chunk * per);
  for (int f0 = 0; f0 < n_frames; f0 += chunk) {
    const int nb = std::min(chunk, n_frames - f0);
    CU(cudaMemcpy2DAsync(d_in.p, row, frames + (size_t)f0 * height * pitch, pitch, row, (size_t)nb * height,
                         frames_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    const uint8_t* img = d_in.p;
    const dim3 blk(32, 8), grd((w + 31) / 32, (h + 7) / 8, nb);
    if (bgr) { bgr_gray_kernel<<<grd, blk, 0, st>>>(d_in.p, width, height, f, d_small.p, w, h); count_launch(); img = d_small.p; }
    else if (scaled) { resize_kernel<<<grd, blk, 0, st>>>(d_in.p, width, height, f, d_small.p, w, h); count_launch(); img = d_small.p; }
    CU(cudaMemsetAsync(d_max.p, 0, nb * sizeof(unsigned), st)); CU(cudaMemsetAsync(d_count.p, 0, nb * sizeof(int), st)); CU(cudaMemsetAsync(d_over.p, 0, nb * sizeof(int), st));
    box_kernel<<<grd, blk, 0, st>>>(img, w, h, d_box.p); count_launch();
    response_kernel<<<grd, blk, 0, st>>>(d_box.p, w, h, d_resp.p, d_max.p); count_launch();
    candidate_kernel<<<dim3((w + kTile - 1) / kTile, (h + kTile - 1) / kTile, nb), 256, 0, st>>>(d_resp.p, w, h, d_max.p, d_cand.p, d_count.p, d_over.p); count_launch();
    GridArgs G{d_cand.p, d_count.p, img, w, h, W, H, d_corner.p, d_spacing.p, d_status.p};
    grid_kernel<<<nb, 32, 0, st>>>(G); count_launch();
    const int nc = nb * (int)per;
    refine_kernel<<<(nc * 32 + 127) / 128, 128, 0, st>>>(img, w, h, (int)per, nc, d_status.p, d_corner.p, d_spacing.p, d_uv.p); count_launch();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(status.data(), d_status.p, nb * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(over.data(), d_over.p, nb * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(uv.data(), d_uv.p, nc * sizeof(double2), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int k = 0; k < nb; ++k) {
      const int fr = f0 + k;
      found[fr] = status[k] == kFound;
      S.candidate_overflow += over[k];
      if (status[k] == kFound) {
        ++S.n_found;
        for (size_t c = 0; c < per; ++c) { uv_out[(fr * per + c) * 2] = uv[k * per + c].x; uv_out[(fr * per + c) * 2 + 1] = uv[k * per + c].y; }
      } else {
        if (status[k] == kNoGrid) ++S.n_no_grid; else if (status[k] == kWrongCount) ++S.n_wrong_count; else ++S.n_no_markers;
      }
    }
  }
  S.gpu_launches = kernel_launch_count() - launches0;
  S.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return ICC_OK;
}

}  // namespace icc
