// Kalibr AprilGrid corner extraction on the GPU (sm_90a): what the reference's extract_board_to_json computes per frame with
// --board_type apriltag, i.e. BoardExtractor::ExtractBoard -> ApriltagDetector::detectTags (third_party/apriltag/apriltag.cpp) on
// the optionally cv::resize'd frame.  The tag math is in icc_aprilgrid_math.cuh; DESIGN.md "AprilGrid corners" has the conventions.
//
// Frames go through in chunks of kChunk (ICC_BOARD_CHUNK_FRAMES overrides it).  Per chunk, every launch covers the whole chunk:
//   resize_kernel      cv::resize INTER_LINEAR (icc_board_math.cuh), skipped at f = 1;
//   tile_kernel        the min and max of every 8 x 8 tile;
//   binarize_kernel    a pixel is dark when the 3 x 3 tiles around its tile span >= kMinContrast grey levels and it is below their
//                      midpoint;
//   erode_kernel       dark pixels whose 4 neighbours are dark start as their own label (this separates the tags from the corner
//                      squares they touch at a point);
//   merge_kernel       4-connected union-find of the dark pixels with atomicMin on the roots (Playne & Hawick, IEEE TPDS 2018);
//   compress_kernel    every dark pixel points at its root, the component's smallest pixel index, and counts itself there;
//   select_kernel      components of at least kMinArea pixels get one of the frame's kMaxQuads slots;
//   extreme_kernel     per component the extreme pixels in 8 directions (64-bit atomicMax on value and pixel index);
//   corner_kernel      one thread per component: of the (up to) 8 extreme pixels, the 4 spanning the largest quadrilateral;
//   edge_kernel        boundary pixels within kEdgeBand of a side add their sub-pixel edge point (where the grey level crosses the
//                      pixel's threshold towards its light neighbour) to that side's fixed-point moments;
//   fit_kernel         one thread per component: a line per side by the moments' principal axis; the corners are their crossings;
//   decode_kernel      one warp per quad: the 12 x 12 model samples and 36 bits through the quad's projective map, the code's
//                      best match among the 587 x 4 codes held in shared memory, and the wrapper's drop reason;
//   frame_kernel       one thread per frame: the wrapper's frame rules; the kept tags' corners are queued for refinement;
//   refine_kernel      one warp per corner of a kept tag: cv::cornerSubPix in FP64 with the wrapper's window and displacement rule.
// Every choice breaks ties on the pixel index and every sum is in integers or in a fixed order, so the result does not depend on
// the chunking or on where the frames came from, except for a frame whose quad slots overflow.
#include "../../include/icc_b200.h"
#include "icc_aprilgrid_math.cuh"
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

using namespace aprilgrid;

constexpr int kChunk = 16;
constexpr int kTile = 8;
constexpr int kMinContrast = 20;     // grey levels between the darkest and the lightest pixel of the 24 x 24 neighbourhood
constexpr int kMinArea = 24;         // pixels of a dark component
constexpr int kMaxQuads = 1024;      // components per frame
constexpr double kMinSide = 10.0;    // px: one pixel per cell
constexpr double kEdgeBand = 2.5;    // px: boundary points within this distance of a side belong to it
constexpr int kFix = 256;            // edge points in 1/256 px

__device__ const uint64_t kDeviceCodes[kTag36h11Count] = {ICC_TAG36H11_CODES};

struct Quad {
  int frame, root, area, status;     // status: 0 candidate, 1 fitted, 2 not a quad
  unsigned long long ext[8];         // (value << 32) | (0xffffffff - pixel index in frame): extreme pixels in 8 directions
  long long mom[4][6];               // per side, edge points in 1/kFix px relative to corner q0: n, sx, sy, sxx, sxy, syy
  int ox, oy;                        // the moments' origin (pixel)
  double q[8];                       // corners, in the quad frame's order (negative shoelace sum)
  double perimeter;
  int id, hamming, rot, drop;        // decode result; drop: kDropNone .. kDropIdRange, -1 not decoded
};

__global__ void resize_kernel(const uint8_t* __restrict__ src, int sw, int sh, double f, uint8_t* __restrict__ dst, int dw, int dh) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= dw || y >= dh) return;
  dst[((size_t)n * dh + y) * dw + x] = board::resize_pixel(src + (size_t)n * sw * sh, sw, sw, sh, f, x, y);
}

__global__ void tile_kernel(const uint8_t* __restrict__ img, int w, int h, int tw, int th, uint8_t* __restrict__ tmin, uint8_t* __restrict__ tmax) {
  const int tx = blockIdx.x * blockDim.x + threadIdx.x, ty = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (tx >= tw || ty >= th) return;
  const uint8_t* I = img + (size_t)n * w * h;
  int lo = 255, hi = 0;
  for (int y = ty * kTile; y < min(h, ty * kTile + kTile); ++y)
    for (int x = tx * kTile; x < min(w, tx * kTile + kTile); ++x) { const int v = I[(size_t)y * w + x]; lo = min(lo, v); hi = max(hi, v); }
  tmin[((size_t)n * th + ty) * tw + tx] = (uint8_t)lo; tmax[((size_t)n * th + ty) * tw + tx] = (uint8_t)hi;
}

// the local threshold 2 T = min + max of the 3 x 3 tiles around pixel (x, y); false where the contrast is below kMinContrast
ICC_D bool local_threshold2(const uint8_t* tmin, const uint8_t* tmax, int tw, int th, int x, int y, int& t2) {
  const int cx = x / kTile, cy = y / kTile;
  int lo = 255, hi = 0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      const int u = min(max(cx + dx, 0), tw - 1), v = min(max(cy + dy, 0), th - 1);
      lo = min(lo, (int)tmin[v * tw + u]); hi = max(hi, (int)tmax[v * tw + u]);
    }
  t2 = lo + hi;
  return hi - lo >= kMinContrast;
}

__global__ void binarize_kernel(const uint8_t* __restrict__ img, int w, int h, int tw, int th, const uint8_t* __restrict__ tmin,
                                const uint8_t* __restrict__ tmax, uint8_t* __restrict__ dark) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= w || y >= h) return;
  const size_t p = ((size_t)n * h + y) * w + x;
  int t2;
  dark[p] = local_threshold2(tmin + (size_t)n * tw * th, tmax + (size_t)n * tw * th, tw, th, x, y, t2) && 2 * (int)img[p] < t2;
}

// a dark pixel stays dark when its four neighbours are dark: at a tag corner the tag and Kalibr's corner square meet at a point,
// and a rotated grid puts two 4-adjacent, mostly dark pixels across it that would join every tag of the grid into one component
__global__ void erode_kernel(int w, int h, const uint8_t* __restrict__ dark, int* __restrict__ label) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= w || y >= h) return;
  const size_t p = ((size_t)n * h + y) * w + x;
  const bool in = x > 0 && y > 0 && x < w - 1 && y < h - 1 && dark[p] && dark[p - 1] && dark[p + 1] && dark[p - w] && dark[p + w];
  label[p] = in ? (int)p : -1;
}

ICC_D int find_root(const int* L, int x) { int y; while ((y = L[x]) != x) x = y; return x; }

ICC_D void unite(int* L, int a, int b) {
  bool done;
  do {
    a = find_root(L, a); b = find_root(L, b);
    if (a < b) { const int old = atomicMin(L + b, a); done = old == b; b = old; }
    else if (b < a) { const int old = atomicMin(L + a, b); done = old == a; a = old; }
    else done = true;
  } while (!done);
}

__global__ void merge_kernel(int w, int h, int* __restrict__ label) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= w || y >= h) return;
  const int p = (int)(((size_t)n * h + y) * w + x);
  if (label[p] < 0) return;
  if (x > 0 && label[p - 1] >= 0) unite(label, p, p - 1);
  if (y > 0 && label[p - w] >= 0) unite(label, p, p - w);
}

__global__ void compress_kernel(int n_px, int* __restrict__ label, int* __restrict__ area) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_px || label[p] < 0) return;
  const int r = find_root(label, p);
  label[p] = r;
  atomicAdd(area + r, 1);
}

// area[root] becomes -(slot + 2) for a selected component (a global quad index), and stays >= 0 otherwise
__global__ void select_kernel(int n_px, int px_per_frame, const int* __restrict__ label, int* __restrict__ area, Quad* __restrict__ quads,
                              int* __restrict__ nquad, int* __restrict__ overflow) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_px || label[p] != p || area[p] < kMinArea) return;
  const int n = p / px_per_frame;
  const int slot = atomicAdd(nquad + n, 1);
  if (slot >= kMaxQuads) { atomicAdd(overflow + n, 1); return; }
  const int g = n * kMaxQuads + slot;
  Quad& Q = quads[g];
  Q.frame = n; Q.root = p; Q.area = area[p]; Q.status = 0; Q.drop = -1;
  area[p] = -(g + 2);
}

ICC_D int quad_of(const int* label, const int* area, int p) {
  const int r = label[p];
  if (r < 0) return -1;
  const int a = area[r];
  return a <= -2 ? -a - 2 : -1;
}

// directions k = 0..7 at 45-degree steps in pixel coordinates: x, x + y, y, y - x, -x, -x - y, -y, x - y
ICC_D int direction_value(int k, int x, int y) {
  switch (k) { case 0: return x; case 1: return x + y; case 2: return y; case 3: return y - x; case 4: return -x; case 5: return -x - y; case 6: return -y; default: return x - y; }
}

__global__ void extreme_kernel(int w, int h, const int* __restrict__ label, const int* __restrict__ area, Quad* __restrict__ quads) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x >= w || y >= h) return;
  const int p = (int)(((size_t)n * h + y) * w + x);
  const int g = quad_of(label, area, p);
  if (g < 0) return;
  const unsigned idx = 0xffffffffu - (unsigned)(y * w + x);
  for (int k = 0; k < 8; ++k) atomicMax(&quads[g].ext[k], ((unsigned long long)(unsigned)(direction_value(k, x, y) + (1 << 20)) << 32) | idx);
}

ICC_D double shoelace(const double* q) {
  double s = 0;
  for (int i = 0; i < 4; ++i) { const int j = (i + 1) & 3; s += q[2 * i] * q[2 * j + 1] - q[2 * j] * q[2 * i + 1]; }
  return s;
}

// put q in the quad frame's winding (negative shoelace sum), starting from the corner the input starts with
ICC_D void wind(double* q) {
  if (shoelace(q) > 0) { double t0 = q[2], t1 = q[3]; q[2] = q[6]; q[3] = q[7]; q[6] = t0; q[7] = t1; }
}

__global__ void corner_kernel(const int* __restrict__ nquad, int w, Quad* __restrict__ quads, int n_frames) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_frames * kMaxQuads || g % kMaxQuads >= min(nquad[g / kMaxQuads], kMaxQuads)) return;
  Quad& Q = quads[g];
  double P[16];
  for (int k = 0; k < 8; ++k) {
    const unsigned pi = 0xffffffffu - (unsigned)(Q.ext[k] & 0xffffffffu);
    P[2 * k] = (double)(pi % w); P[2 * k + 1] = (double)(pi / w);
  }
  // the 4 of the 8 support points (in boundary order) with the largest area
  double best = -1; int bi[4] = {0, 2, 4, 6};
  for (int a = 0; a < 8; ++a)
    for (int b = a + 1; b < 8; ++b)
      for (int c = b + 1; c < 8; ++c)
        for (int d = c + 1; d < 8; ++d) {
          const double q[8] = {P[2 * a], P[2 * a + 1], P[2 * b], P[2 * b + 1], P[2 * c], P[2 * c + 1], P[2 * d], P[2 * d + 1]};
          const double s = fabs(shoelace(q));
          if (s > best) { best = s; bi[0] = a; bi[1] = b; bi[2] = c; bi[3] = d; }
        }
  for (int i = 0; i < 4; ++i) { Q.q[2 * i] = P[2 * bi[i]]; Q.q[2 * i + 1] = P[2 * bi[i] + 1]; }
  wind(Q.q);
  Q.ox = (int)Q.q[0]; Q.oy = (int)Q.q[1];
  double mind = 1e30;
  for (int i = 0; i < 4; ++i) { const int j = (i + 1) & 3; mind = fmin(mind, hypot(Q.q[2 * j] - Q.q[2 * i], Q.q[2 * j + 1] - Q.q[2 * i + 1])); }
  // a tag's component fills at least its 2-cell border ring, 64 % of the quad
  Q.status = (mind >= kMinSide && Q.area >= 0.4 * 0.5 * best) ? 1 : 2;
}

__global__ void edge_kernel(const uint8_t* __restrict__ img, int w, int h, int tw, int th, const uint8_t* __restrict__ tmin, const uint8_t* __restrict__ tmax,
                            const int* __restrict__ label, const int* __restrict__ area, Quad* __restrict__ quads) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (x < 1 || y < 1 || x >= w - 1 || y >= h - 1) return;
  const size_t p = ((size_t)n * h + y) * w + x;
  const int g = quad_of(label, area, (int)p);
  if (g < 0) return;
  Quad& Q = quads[g];
  if (Q.status != 1) return;
  // the edge point: towards each 4-neighbour outside the (eroded) component, where the grey level first crosses this pixel's
  // threshold within two pixels
  const uint8_t* I = img + (size_t)n * w * h;
  int t2;
  local_threshold2(tmin + (size_t)n * tw * th, tmax + (size_t)n * tw * th, tw, th, x, y, t2);
  const double T = 0.5 * t2;
  double ex = 0, ey = 0; int ne = 0;
  const int dx[4] = {1, -1, 0, 0}, dy[4] = {0, 0, 1, -1};
  for (int k = 0; k < 4; ++k) {
    if (label[(int)p + dx[k] + dy[k] * w] >= 0) continue;
    const int x2 = min(max(x + 2 * dx[k], 0), w - 1), y2 = min(max(y + 2 * dy[k], 0), h - 1);
    const double v0 = I[(size_t)y * w + x], v1 = I[(size_t)(y + dy[k]) * w + x + dx[k]], v2 = I[(size_t)y2 * w + x2];
    double t;
    if (v0 >= T) t = 0.0;
    else if (v1 >= T) t = (T - v0) / (v1 - v0);
    else if (v2 > v1 && v2 >= T) t = 1.0 + (T - v1) / (v2 - v1);
    else continue;
    ex += x + t * dx[k]; ey += y + t * dy[k]; ++ne;
  }
  if (!ne) return;
  ex /= ne; ey /= ne;
  // the side it lies on: within kEdgeBand of the chord, away from the corners
  for (int i = 0; i < 4; ++i) {
    const int j = (i + 1) & 3;
    const double ax = Q.q[2 * i], ay = Q.q[2 * i + 1], bx = Q.q[2 * j] - ax, by = Q.q[2 * j + 1] - ay;
    const double L2 = bx * bx + by * by, t = ((ex - ax) * bx + (ey - ay) * by) / L2;
    if (t < 0.1 || t > 0.9) continue;
    const double d = fabs((ex - ax) * by - (ey - ay) * bx) / sqrt(L2);
    if (d > kEdgeBand) continue;
    const long long fx = llrint((ex - Q.ox) * kFix), fy = llrint((ey - Q.oy) * kFix);
    long long* m = Q.mom[i];
    atomicAdd((unsigned long long*)&m[0], 1ull);
    atomicAdd((unsigned long long*)&m[1], (unsigned long long)fx); atomicAdd((unsigned long long*)&m[2], (unsigned long long)fy);
    atomicAdd((unsigned long long*)&m[3], (unsigned long long)(fx * fx)); atomicAdd((unsigned long long*)&m[4], (unsigned long long)(fx * fy));
    atomicAdd((unsigned long long*)&m[5], (unsigned long long)(fy * fy));
    break;
  }
}

__global__ void fit_kernel(const int* __restrict__ nquad, Quad* __restrict__ quads, int n_frames) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_frames * kMaxQuads || g % kMaxQuads >= min(nquad[g / kMaxQuads], kMaxQuads)) return;
  Quad& Q = quads[g];
  if (Q.status != 1) return;
  double L[4][3];   // a x + b y = c, (a, b) unit
  for (int i = 0; i < 4; ++i) {
    const long long* m = Q.mom[i];
    if (m[0] < 3) { Q.status = 2; return; }
    const double nn = (double)m[0], mx = m[1] / nn, my = m[2] / nn;
    const double cxx = m[3] / nn - mx * mx, cxy = m[4] / nn - mx * my, cyy = m[5] / nn - my * my;
    // the normal is the eigenvector of the smaller eigenvalue of the scatter
    const double ang = 0.5 * atan2(2 * cxy, cxx - cyy);
    const double a = -sin(ang), b = cos(ang);
    L[i][0] = a; L[i][1] = b; L[i][2] = a * (mx / kFix + Q.ox) + b * (my / kFix + Q.oy);
  }
  double q[8];
  for (int i = 0; i < 4; ++i) {   // corner i is where side i - 1 meets side i
    const double* A = L[(i + 3) & 3]; const double* B = L[i];
    const double det = A[0] * B[1] - A[1] * B[0];
    if (fabs(det) < 1e-6) { Q.status = 2; return; }
    q[2 * i] = (A[2] * B[1] - A[1] * B[2]) / det;
    q[2 * i + 1] = (A[0] * B[2] - A[2] * B[0]) / det;
    if (hypot(q[2 * i] - Q.q[2 * i], q[2 * i + 1] - Q.q[2 * i + 1]) > 4.0 + 0.1 * sqrt(fabs(shoelace(Q.q)))) { Q.status = 2; return; }
  }
  double per = 0;
  for (int i = 0; i < 4; ++i) { const int j = (i + 1) & 3; per += hypot(q[2 * j] - q[2 * i], q[2 * j + 1] - q[2 * i + 1]); }
  if (!(shoelace(q) < 0)) { Q.status = 2; return; }
  for (int k = 0; k < 8; ++k) Q.q[k] = q[k];
  Q.perimeter = per;
}

ICC_D double warp_sum(double v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) decode_kernel(const uint8_t* __restrict__ img, int w, int h, const int* __restrict__ nquad, Quad* __restrict__ quads, int n_frames) {
  __shared__ uint64_t codes[kTag36h11Count];
  for (int i = threadIdx.x; i < kTag36h11Count; i += blockDim.x) codes[i] = kDeviceCodes[i];
  __syncthreads();
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (g >= n_frames * kMaxQuads || g % kMaxQuads >= min(nquad[g / kMaxQuads], kMaxQuads)) return;
  Quad& Q = quads[g];
  if (Q.status != 1) return;
  const uint8_t* I = img + (size_t)Q.frame * w * h;
  const QuadMap M = quad_map(Q.q);
  double sb[kGraySums], sw[kGraySums];
  for (int k = 0; k < kGraySums; ++k) sb[k] = sw[k] = 0.0;
  for (int k = lane; k < kModelSamples; k += 32) {
    int ix, iy;
    const int kind = model_kind(k, ix, iy);
    if (!kind) continue;
    const double x = (ix + 0.5) / kCells, y = (iy + 0.5) / kCells;
    double v;
    if (!sample_pixel(I, w, w, h, M, x, y, v)) continue;
    gray_add(kind == 2 ? sw : sb, x, y, v);
  }
  for (int k = 0; k < kGraySums; ++k) { sb[k] = warp_sum(sb[k]); sw[k] = warp_sum(sw[k]); }
  double cb[4], cw[4];
  gray_solve(sb, cb); gray_solve(sw, cw);
  uint64_t code = 0; bool bad = false;
  for (int k0 = 0; k0 < kDim * kDim; k0 += 32) {
    const int k = k0 + lane;
    bool one = false, ok = true;
    if (k < kDim * kDim) {
      double x, y, v;
      bit_position(k, x, y);
      ok = sample_pixel(I, w, w, h, M, x, y, v);
      one = ok && v > 0.5 * (gray_eval(cb, x, y) + gray_eval(cw, x, y));
    }
    const unsigned ones = __ballot_sync(0xffffffffu, one);
    bad |= __ballot_sync(0xffffffffu, !ok) != 0;
    for (int j = 0; j < 32 && k0 + j < kDim * kDim; ++j) code = (code << 1) | ((ones >> j) & 1u);
  }
  if (bad) { if (lane == 0) Q.drop = -1; return; }
  int key = decode_key(code, codes, lane, 32);
  for (int o = 16; o; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
  if (lane) return;
  int ham, id, rot;
  unpack_key(key, ham, id, rot);
  double p[8];
  for (int i = 0; i < 4; ++i) { p[2 * i] = Q.q[2 * ((i + rot) & 3)]; p[2 * i + 1] = Q.q[2 * ((i + rot) & 3) + 1]; }
  for (int k = 0; k < 8; ++k) Q.q[k] = p[k];
  Q.id = id; Q.hamming = ham; Q.rot = rot;
  Q.drop = drop_reason(p, ham, id, w, h);
}

struct FrameOut {
  int verdict;                       // kFrameFound / kFrameFewTags / kFrameDuplicate
  int n_border, n_not_good, n_id_range, n_not_decoded;
};

// one thread per frame: the frame rules, and the refinement queue of the kept tags (tag slots in found frames)
__global__ void frame_kernel(const int* __restrict__ nquad, const Quad* __restrict__ quads, int n_frames, int n_tags, FrameOut* __restrict__ fo,
                             int* __restrict__ kept, int* __restrict__ n_kept) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_frames) return;
  FrameOut F{};
  const int nq = min(nquad[n], kMaxQuads);
  int ids[kIdLimit + 1], nk = 0;   // more than kIdLimit kept tags always hold a duplicate
  bool dup = false;
  for (int s = 0; s < nq; ++s) {
    const Quad& Q = quads[n * kMaxQuads + s];
    if (Q.status != 1 || Q.drop < 0) { F.n_not_decoded += Q.status == 1; continue; }
    if (Q.drop == kDropBorder) { ++F.n_border; continue; }
    if (Q.drop == kDropNotGood) { ++F.n_not_good; continue; }
    if (Q.drop == kDropIdRange) { ++F.n_id_range; continue; }
    if (nk <= kIdLimit) ids[nk] = Q.id; else dup = true;
    ++nk;
  }
  F.verdict = dup ? kFrameDuplicate : frame_verdict(min(nk, kIdLimit + 1), ids);
  fo[n] = F;
  if (F.verdict != kFrameFound) return;
  for (int s = 0; s < nq; ++s) {
    const Quad& Q = quads[n * kMaxQuads + s];
    // a tag of the id range without a board point (a board of fewer than 36 tags) counts for the rules but has no slot
    if (Q.status == 1 && Q.drop == kDropNone && Q.id < n_tags) kept[atomicAdd(n_kept, 1)] = n * kMaxQuads + s;
  }
}

// one warp per corner of a queued tag; uv and status are per frame and point id (t << 2) + i
__global__ void __launch_bounds__(128) refine_kernel(const uint8_t* __restrict__ img, int w, int h, const Quad* __restrict__ quads, const int* __restrict__ kept,
                                                     const int* __restrict__ n_kept, int n_points, double2* __restrict__ uv, int* __restrict__ status) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (g >= 4 * *n_kept) return;
  const Quad& Q = quads[kept[g >> 2]];
  const int i = g & 3;
  const uint8_t* I = img + (size_t)Q.frame * w * h;
  const double r = subpix_radius(Q.perimeter);
  const int win = subpix_half_window(r);
  const float sx = (float)Q.q[2 * i], sy = (float)Q.q[2 * i + 1];
  float cx = sx, cy = sy;
  for (int it = 0; it < kSubpixMaxIters; ++it) {
    double s[5] = {0, 0, 0, 0, 0};
    subpix_accumulate(I, w, w, h, cx, cy, win, lane, 32, s);
    for (int k = 0; k < 5; ++k) s[k] = warp_sum(s[k]);
    double err;
    if (!subpix_update(s, cx, cy, err)) break;
    if (cx < 0 || cx >= w || cy < 0 || cy >= h) break;
    if (err <= kSubpixEps * kSubpixEps) break;
  }
  subpix_finish(sx, sy, win, cx, cy);
  if (lane) return;
  const double d2 = ((double)cx - sx) * ((double)cx - sx) + ((double)cy - sy) * ((double)cy - sy);
  const size_t o = (size_t)Q.frame * n_points + Q.id * 4 + i;
  uv[o] = make_double2(cx, cy);
  status[o] = d2 <= r * r ? 1 : -1;
}

}  // namespace

#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status extract_aprilgrid(cudaStream_t st, int n_frames, int width, int height, int64_t pitch, const uint8_t* frames, bool frames_on_device, int tags_x, int tags_y,
                             double f, double* uv_out, int32_t* status_out, int32_t* found, icc_aprilgrid_summary& S, std::string& err) {
  const auto t0 = std::chrono::steady_clock::now();
  const int launches0 = kernel_launch_count();
  memset(&S, 0, sizeof S);
  const bool scaled = f != 1.0;
  const int w = scaled ? board::resize_dim(width, f) : width, h = scaled ? board::resize_dim(height, f) : height;
  S.width = w; S.height = h;
  if (w < 16 || h < 16) { err = "the (downsampled) frame is too small"; return ICC_ERR_INVALID_ARGUMENT; }
  int chunk = kChunk;
  if (const char* e = getenv("ICC_BOARD_CHUNK_FRAMES")) chunk = std::max(1, atoi(e));
  chunk = std::min(chunk, std::max(n_frames, 1));
  if ((double)chunk * w * h >= 2.0e9) chunk = std::max(1, (int)(2.0e9 / ((double)w * h)) - 1);   // int pixel indices
  const int tw = (w + kTile - 1) / kTile, th = (h + kTile - 1) / kTile, n_tags = tags_x * tags_y, np = 4 * n_tags;
  const size_t px = (size_t)w * h;
  DevBuf<uint8_t> d_in, d_small, d_tmin, d_tmax, d_dark; DevBuf<int> d_label, d_area, d_nquad, d_over, d_kept, d_nkept, d_status;
  DevBuf<Quad> d_quads; DevBuf<FrameOut> d_fo; DevBuf<double2> d_uv;
  CU(d_in.alloc(chunk * (size_t)width * height));
  if (scaled) CU(d_small.alloc(chunk * px));
  CU(d_tmin.alloc((size_t)chunk * tw * th)); CU(d_tmax.alloc((size_t)chunk * tw * th));
  CU(d_dark.alloc(chunk * px)); CU(d_label.alloc(chunk * px)); CU(d_area.alloc(chunk * px));
  CU(d_nquad.alloc(chunk)); CU(d_over.alloc(chunk)); CU(d_kept.alloc((size_t)chunk * kMaxQuads)); CU(d_nkept.alloc(1));
  CU(d_quads.alloc((size_t)chunk * kMaxQuads)); CU(d_fo.alloc(chunk)); CU(d_uv.alloc((size_t)chunk * np)); CU(d_status.alloc((size_t)chunk * np));
  std::vector<FrameOut> fo(chunk);
  std::vector<int> over(chunk), nquad(chunk), status((size_t)chunk * np);
  std::vector<double2> uv((size_t)chunk * np);
  for (int f0 = 0; f0 < n_frames; f0 += chunk) {
    const int nb = std::min(chunk, n_frames - f0);
    const int n_px = nb * (int)px;
    CU(cudaMemcpy2DAsync(d_in.p, width, frames + (size_t)f0 * height * pitch, pitch, width, (size_t)nb * height,
                         frames_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    const uint8_t* img = d_in.p;
    const dim3 blk(32, 8), grd((w + 31) / 32, (h + 7) / 8, nb);
    if (scaled) { resize_kernel<<<grd, blk, 0, st>>>(d_in.p, width, height, f, d_small.p, w, h); count_launch(); img = d_small.p; }
    CU(cudaMemsetAsync(d_area.p, 0, (size_t)n_px * sizeof(int), st)); CU(cudaMemsetAsync(d_nquad.p, 0, nb * sizeof(int), st));
    CU(cudaMemsetAsync(d_over.p, 0, nb * sizeof(int), st)); CU(cudaMemsetAsync(d_nkept.p, 0, sizeof(int), st));
    CU(cudaMemsetAsync(d_quads.p, 0, (size_t)nb * kMaxQuads * sizeof(Quad), st));
    CU(cudaMemsetAsync(d_uv.p, 0xff, (size_t)nb * np * sizeof(double2), st)); CU(cudaMemsetAsync(d_status.p, 0, (size_t)nb * np * sizeof(int), st));
    tile_kernel<<<dim3((tw + 15) / 16, (th + 15) / 16, nb), dim3(16, 16), 0, st>>>(img, w, h, tw, th, d_tmin.p, d_tmax.p); count_launch();
    binarize_kernel<<<grd, blk, 0, st>>>(img, w, h, tw, th, d_tmin.p, d_tmax.p, d_dark.p); count_launch();
    erode_kernel<<<grd, blk, 0, st>>>(w, h, d_dark.p, d_label.p); count_launch();
    merge_kernel<<<grd, blk, 0, st>>>(w, h, d_label.p); count_launch();
    compress_kernel<<<(n_px + 255) / 256, 256, 0, st>>>(n_px, d_label.p, d_area.p); count_launch();
    select_kernel<<<(n_px + 255) / 256, 256, 0, st>>>(n_px, (int)px, d_label.p, d_area.p, d_quads.p, d_nquad.p, d_over.p); count_launch();
    extreme_kernel<<<grd, blk, 0, st>>>(w, h, d_label.p, d_area.p, d_quads.p); count_launch();
    const int nq = nb * kMaxQuads;
    corner_kernel<<<(nq + 127) / 128, 128, 0, st>>>(d_nquad.p, w, d_quads.p, nb); count_launch();
    edge_kernel<<<grd, blk, 0, st>>>(img, w, h, tw, th, d_tmin.p, d_tmax.p, d_label.p, d_area.p, d_quads.p); count_launch();
    fit_kernel<<<(nq + 127) / 128, 128, 0, st>>>(d_nquad.p, d_quads.p, nb); count_launch();
    decode_kernel<<<(nq * 32 + 255) / 256, 256, 0, st>>>(img, w, h, d_nquad.p, d_quads.p, nb); count_launch();
    frame_kernel<<<(nb + 63) / 64, 64, 0, st>>>(d_nquad.p, d_quads.p, nb, n_tags, d_fo.p, d_kept.p, d_nkept.p); count_launch();
    refine_kernel<<<(nq * 4 * 32 + 127) / 128, 128, 0, st>>>(img, w, h, d_quads.p, d_kept.p, d_nkept.p, np, d_uv.p, d_status.p); count_launch();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(fo.data(), d_fo.p, nb * sizeof(FrameOut), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(over.data(), d_over.p, nb * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(nquad.data(), d_nquad.p, nb * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(uv.data(), d_uv.p, (size_t)nb * np * sizeof(double2), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(status.data(), d_status.p, (size_t)nb * np * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int k = 0; k < nb; ++k) {
      const size_t fr = (size_t)f0 + k;
      const FrameOut& F = fo[k];
      found[fr] = F.verdict == kFrameFound;
      S.n_quads += std::min(nquad[k], kMaxQuads); S.quad_overflow += over[k];
      S.n_not_decoded += F.n_not_decoded; S.n_border += F.n_border; S.n_not_good += F.n_not_good; S.n_id_range += F.n_id_range;
      if (F.verdict == kFrameFound) ++S.n_found; else if (F.verdict == kFrameFewTags) ++S.n_few_tags; else ++S.n_duplicate;
      for (int c = 0; c < np; ++c) {
        const int s = status[k * np + c];
        status_out[fr * np + c] = s;
        uv_out[(fr * np + c) * 2] = uv[k * np + c].x; uv_out[(fr * np + c) * 2 + 1] = uv[k * np + c].y;
        S.n_corners_kept += s == 1; S.n_corners_moved += s == -1;
      }
    }
  }
  S.gpu_launches = kernel_launch_count() - launches0;
  S.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return ICC_OK;
}

}  // namespace icc
