// Static multi-pose IMU intrinsic calibration (sm_90a): the step that produces the hot CLI's `--imu_intrinsics` file.
//
// Replaces what the reference runs serially on the CPU in
//   StaticImuCalibrator::CalibrateAcc / CalibrateAccGyro     src/core/static_imu_calibrator.cc:54-186, :188-337
//   DataInterval::InitialInterval / TimeToIndex               include/OpenCameraCalibrator/utils/imu_data_interval.h
//   DataMean / DataVariance / StaticIntervalsDetector / ExtractIntervalsSamples    src/utils/imu_data_interval.cc
// The reference recomputes a 101-sample windowed variance at every sample once per threshold multiplier (ten passes) and
// re-integrates every rotation between static poses with RK4 under autodiff Jets on every LM evaluation.  Here:
//   * one kernel, one thread per sample, computes the windowed variance norm ONCE from a shared-memory window; the ten multipliers
//     differ only in the comparison.  The arithmetic is the reference's sequential two-pass loop with explicitly rounded operations
//     (no FMA contraction), so every threshold decision equals the CPU's bit for bit;
//   * static intervals of all ten multipliers = runs of the ten boolean sequences: run starts / ends are flag changes, compacted
//     with warp ballots and a block-count prefix scan (no host walk over samples);
//   * the ten accelerometer problems run concurrently, one CTA each, the whole trust-region loop inside the kernel (closed-form
//     Jacobian rows, block-reduced 9x9 normal equations, one-thread damped solve and acceptance logic);
//   * the gyroscope residual of a transition is normalize(A_{n-1} ... A_0 e0) (icc_static_imu_math.cuh): one CTA per transition,
//     16 sample chunks x 16 parameter directions, each thread multiplies its chunk's dual 4x4 matrices, then a tree over the chunks.
//     The 9-12 unknown LM runs on the host with one small readback per iteration (like icc_camcal.cu's driver).
#include "../../include/icc_b200.h"
#include "icc_device_math.cuh"
#include "icc_host.h"
#include "icc_reduce.cuh"
#include "icc_static_imu_math.cuh"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace icc {

namespace {

using simu::Dual;
using simu::LmState;

constexpr int kMult = 10;          // threshold multipliers 1..10 (static_imu_calibrator.cc:83)
constexpr int kThreads = 256;
constexpr int kChunks = 16, kDirs = 16;   // gyroscope kernel: sample chunks x parameter directions = 256 threads

ICC_D unsigned lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }

// DataVariance(samples, [i-h, i+h]).norm() (imu_data_interval.cc:38-53) for every i in [h, n-h): sequential two-pass sums in the
// reference's order, every operation rounded on its own (__dadd_rn / __dmul_rn cannot be contracted into FMAs).
__global__ void __launch_bounds__(kThreads) window_norm_kernel(int n, int h, const double* __restrict__ acc, int stage, double* __restrict__ norm) {
  extern __shared__ double win[];
  const int c0 = h + blockIdx.x * blockDim.x;             // first window centre of this block
  const int i = c0 + threadIdx.x;
  const double* src = acc;
  int base = 0;
  if (stage) {
    const int lo = c0 - h, hi = min(c0 + (int)blockDim.x + h, n);
    for (int k = lo + threadIdx.x; k < hi; k += blockDim.x) { win[3 * (k - lo)] = acc[3 * (size_t)k]; win[3 * (k - lo) + 1] = acc[3 * (size_t)k + 1]; win[3 * (k - lo) + 2] = acc[3 * (size_t)k + 2]; }
    __syncthreads();
    src = win; base = lo;
  }
  if (i >= n - h) return;
  const int w = 2 * h + 1;
  double m0 = 0.0, m1 = 0.0, m2 = 0.0;
  for (int k = i - h; k <= i + h; ++k) {
    const double* x = src + 3 * (size_t)(k - base);
    m0 = __dadd_rn(m0, x[0]); m1 = __dadd_rn(m1, x[1]); m2 = __dadd_rn(m2, x[2]);
  }
  const double nd = (double)w;
  m0 = __ddiv_rn(m0, nd); m1 = __ddiv_rn(m1, nd); m2 = __ddiv_rn(m2, nd);
  double v0 = 0.0, v1 = 0.0, v2 = 0.0;
  for (int k = i - h; k <= i + h; ++k) {
    const double* x = src + 3 * (size_t)(k - base);
    const double d0 = __dsub_rn(x[0], m0), d1 = __dsub_rn(x[1], m1), d2 = __dsub_rn(x[2], m2);
    v0 = __dadd_rn(v0, __dmul_rn(d0, d0)); v1 = __dadd_rn(v1, __dmul_rn(d1, d1)); v2 = __dadd_rn(v2, __dmul_rn(d2, d2));
  }
  const double nm1 = (double)(w - 1);
  v0 = __ddiv_rn(v0, nm1); v1 = __ddiv_rn(v1, nm1); v2 = __ddiv_rn(v2, nm1);
  norm[i] = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v0, v0), __dmul_rn(v1, v1)), __dmul_rn(v2, v2)));   // Eigen: (x^2 + y^2) + z^2
}

struct RunArgs {
  int n, h, nb, cap;
  const double* norm;
  double thr[kMult];           // th_mult * norm_th, rounded as on the host
  int* counts;                 // [2][kMult][nb]: starts / ends per block
  const int* offsets;          // same layout, exclusive prefix over blocks (write pass)
  int* starts; int* ends;      // [kMult][cap]
};

// bit m-1 set where window centre j is static under multiplier m (`norm < threshold`, imu_data_interval.cc:123-134)
ICC_D unsigned static_bits(const RunArgs& A, int j) {
  if (j < A.h || j >= A.n - A.h) return 0u;
  const double v = A.norm[j];
  unsigned b = 0u;
#pragma unroll
  for (int m = 0; m < kMult; ++m) b |= (v < A.thr[m]) ? (1u << m) : 0u;
  return b;
}

// StaticIntervalsDetector's state machine == runs of the boolean sequence: a start where the flag turns on, an end (inclusive) where
// it turns off at the next centre or the scan ends (the interval still open at the end closes at n-h-1, :138-143).
// write == 0: per-block counts; write == 1: scatter to the prefix-scanned positions.
__global__ void __launch_bounds__(kThreads) runs_kernel(RunArgs A, int write) {
  __shared__ int wcount[2][kMult][kThreads / 32];
  const int i = A.h + blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned f = static_bits(A, i);
  const unsigned st = f & ~static_bits(A, i - 1), en = f & ~static_bits(A, i + 1);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  unsigned bal[2][kMult];
#pragma unroll
  for (int m = 0; m < kMult; ++m) {
    bal[0][m] = __ballot_sync(0xffffffffu, (st >> m) & 1u);
    bal[1][m] = __ballot_sync(0xffffffffu, (en >> m) & 1u);
    if (lane == 0) { wcount[0][m][warp] = __popc(bal[0][m]); wcount[1][m][warp] = __popc(bal[1][m]); }
  }
  __syncthreads();
  if (!write) {
    if (threadIdx.x < 2 * kMult) {
      const int k = threadIdx.x / kMult, m = threadIdx.x % kMult;
      int s = 0; for (int w = 0; w < nw; ++w) s += wcount[k][m][w];
      A.counts[((size_t)k * kMult + m) * A.nb + blockIdx.x] = s;
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int m = 0; m < kMult; ++m) {
      if (!((bal[k][m] >> lane) & 1u)) continue;
      int pos = A.offsets[((size_t)k * kMult + m) * A.nb + blockIdx.x] + __popc(bal[k][m] & lanemask_lt());
      for (int w = 0; w < warp; ++w) pos += wcount[k][m][w];
      (k == 0 ? A.starts : A.ends)[(size_t)m * A.cap + pos] = i;
    }
}

// exclusive prefix over the blocks of one (kind, multiplier) row; totals[row] = its sum
__global__ void __launch_bounds__(kThreads) block_scan_kernel(int nb, const int* __restrict__ counts, int* __restrict__ offsets, int* __restrict__ totals) {
  __shared__ int part[kThreads];
  const int row = blockIdx.x;
  const int* c = counts + (size_t)row * nb;
  int* o = offsets + (size_t)row * nb;
  const int per = (nb + blockDim.x - 1) / blockDim.x, b0 = threadIdx.x * per, b1 = min(nb, b0 + per);
  int s = 0; for (int b = b0; b < b1; ++b) s += c[b];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) { int acc = 0; for (int t = 0; t < (int)blockDim.x; ++t) { const int v = part[t]; part[t] = acc; acc += v; } totals[row] = acc; }
  __syncthreads();
  int run = part[threadIdx.x];
  for (int b = b0; b < b1; ++b) { o[b] = run; run += c[b]; }
}

// ExtractIntervalsSamples' filter (imu_data_interval.cc:62-76): keep the intervals with at least `ns` samples, in order.  One CTA
// per multiplier, ballot compaction.
__global__ void __launch_bounds__(kThreads) keep_kernel(int cap, int ns, const int* __restrict__ totals, const int* __restrict__ starts, const int* __restrict__ ends,
                                                        int* __restrict__ kept_s, int* __restrict__ kept_e, int* __restrict__ kept_n) {
  __shared__ int wc[kThreads / 32];
  __shared__ int base;
  const int m = blockIdx.x, nr = totals[m];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int r0 = 0; r0 < nr; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    const int s = r < nr ? starts[(size_t)m * cap + r] : 0, e = r < nr ? ends[(size_t)m * cap + r] : -1;
    const bool keep = r < nr && e - s + 1 >= ns;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wc[warp] = __popc(b);
    __syncthreads();
    int pos = base + __popc(b & lanemask_lt()), tot = 0;
    for (int w = 0; w < nw; ++w) { if (w < warp) pos += wc[w]; tot += wc[w]; }
    if (keep) { kept_s[(size_t)m * cap + pos] = s; kept_e[(size_t)m * cap + pos] = e; }
    __syncthreads();
    if (threadIdx.x == 0) base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) kept_n[m] = base;
}

struct AccTriad { double ms[9], b[3]; };

// DataMean over each kept interval (sequential sum, then / n; imu_data_interval.cc:25-36), optionally of the calibrated samples
// ms (x - b) with ms = T K of the accelerometer triad (UnbiasNormalize, types.h:293-296; CalibrateAccGyro :197-203)
__global__ void interval_mean_kernel(int nk, const int2* __restrict__ iv, const double* __restrict__ x, int calibrated, AccTriad tri, double* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nk) return;
  const int s = iv[k].x, e = iv[k].y;
  double m0 = 0.0, m1 = 0.0, m2 = 0.0;
  for (int j = s; j <= e; ++j) {
    double a0 = x[3 * (size_t)j], a1 = x[3 * (size_t)j + 1], a2 = x[3 * (size_t)j + 2];
    if (calibrated) {
      const double u0 = a0 - tri.b[0], u1 = a1 - tri.b[1], u2 = a2 - tri.b[2];
      a0 = tri.ms[0] * u0 + tri.ms[1] * u1 + tri.ms[2] * u2; a1 = tri.ms[3] * u0 + tri.ms[4] * u1 + tri.ms[5] * u2; a2 = tri.ms[6] * u0 + tri.ms[7] * u1 + tri.ms[8] * u2;
    }
    m0 += a0; m1 += a1; m2 += a2;
  }
  const double nd = (double)(e - s + 1);
  out[3 * k] = m0 / nd; out[3 * k + 1] = m1 / nd; out[3 * k + 2] = m2 / nd;
}

struct AccFitArgs {
  const double* acc;       // raw samples
  const int2* kept;        // kept intervals of all multipliers, concatenated
  const double* means;     // their raw means (acc_use_means)
  int koff[kMult + 1];
  int fit[kMult];          // multiplier has enough intervals
  int ns, use_means;
  double g_mag;
  double x0[9];
  TrOptions o;
  double* out;             // per multiplier: x[9], initial cost, final cost, iterations, termination, successful steps
};
constexpr int kAccOut = 14, kSums = normal_equation_sums(9);

// cost, J^T J, J^T r of one multiplier's problem at x, reduced over the block in a fixed order; valid in thread 0
ICC_D void acc_normal_equations(const AccFitArgs& A, int m, const double* x, double (*red)[kSums], double* tot) {
  double s[kSums];
#pragma unroll
  for (int k = 0; k < kSums; ++k) s[k] = 0.0;
  const int k0 = A.koff[m], nk = A.koff[m + 1] - k0;
  const int nsamp = A.use_means ? nk : nk * A.ns;
  for (int j = threadIdx.x; j < nsamp; j += blockDim.x) {
    double a[3];
    if (A.use_means) { a[0] = A.means[3 * (k0 + j)]; a[1] = A.means[3 * (k0 + j) + 1]; a[2] = A.means[3 * (k0 + j) + 2]; }
    else { const size_t q = (size_t)A.kept[k0 + j / A.ns].x + j % A.ns; a[0] = A.acc[3 * q]; a[1] = A.acc[3 * q + 1]; a[2] = A.acc[3 * q + 2]; }
    double J[9];
    const double r = simu::acc_residual(x, a, A.g_mag, J);
    normal_equation_row<9>(s, J, r);
  }
  block_sums<kSums>(s, red, tot);
}

// one CTA per threshold multiplier: CalibrateAcc's ceres::Solve (static_imu_calibrator.cc:113-130) entirely on the device
__global__ void __launch_bounds__(kThreads) acc_fit_kernel(AccFitArgs A) {
  __shared__ double red[kThreads / 32][kSums];
  __shared__ double tot[kSums];
  __shared__ double x[12];
  __shared__ LmState L;
  __shared__ int go;
  const int m = blockIdx.x;
  if (!A.fit[m]) return;
  if (threadIdx.x < 12) x[threadIdx.x] = threadIdx.x < 9 ? A.x0[threadIdx.x] : 0.0;
  __syncthreads();
  acc_normal_equations(A, m, x, red, tot);
  if (threadIdx.x == 0) {
    double H[12][12], g[12], c; unpack_normal_equations<9, 12>(tot, H, g, c);
    simu::lm_start(L, A.o, 9, x, c, H, g);
  }
  for (;;) {
    if (threadIdx.x == 0) { go = simu::lm_propose(L) ? 1 : 0; for (int p = 0; p < 9; ++p) x[p] = L.xc[p]; }
    __syncthreads();
    if (!go) break;
    acc_normal_equations(A, m, x, red, tot);
    if (threadIdx.x == 0) { double H[12][12], g[12], c; unpack_normal_equations<9, 12>(tot, H, g, c); simu::lm_consider(L, c, H, g); }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* o = A.out + (size_t)m * kAccOut;
    for (int p = 0; p < 9; ++p) o[p] = L.x[p];
    o[9] = L.T.initial_cost; o[10] = L.T.cost; o[11] = L.T.iterations; o[12] = L.T.termination; o[13] = L.T.successful;
  }
}

__global__ void unbias_kernel(int n, const double* __restrict__ g, double b0, double b1, double b2, double* __restrict__ out) {   // Unbias (types.h:299-302)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[3 * (size_t)i] = g[3 * (size_t)i] - b0; out[3 * (size_t)i + 1] = g[3 * (size_t)i + 1] - b1; out[3 * (size_t)i + 2] = g[3 * (size_t)i + 2] - b2;
}

struct GyroArgs {
  const double* x;        // unbiased gyroscope samples
  const double* t;
  const int2* span;       // per transition: first / last gyroscope sample (static_imu_calibrator.cc:261-279)
  const double* g01;      // per transition: unit gravity of pose i, pose i+1 (6)
  double gyro_dt;
  double p[12];
  int np, with_bias;
  double* out;            // per transition: r[3], then J[3][12] row-major
};
constexpr int kGyroOut = 3 + 3 * 12;

// MultiPosGyroResidual of one transition and its Jacobian (all directions at once)
__global__ void __launch_bounds__(kChunks * kDirs) gyro_eval_kernel(GyroArgs G) {
  __shared__ Dual park[kChunks / 2][kDirs][16];
  const int tr = blockIdx.x, c = threadIdx.x / kDirs, d = threadIdx.x % kDirs;
  Dual p[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) p[j] = simu::dual(G.p[j], j == d ? 1.0 : 0.0);
  const int i0 = G.span[tr].x, i1 = G.span[tr].y, m = i1 - i0, L = (m + kChunks - 1) / kChunks;
  const int k0 = min(i1, i0 + c * L), k1 = min(i1, i0 + (c + 1) * L);
  Dual P[16];
  simu::chain_product(p, G.with_bias != 0, G.x, G.t, G.gyro_dt, k0, k1, P);
  for (int s = 1; s < kChunks; s <<= 1) {          // (P_later, D_later) o (P, D), pairwise over the chunks
    if ((c & (2 * s - 1)) == s) for (int k = 0; k < 16; ++k) park[c / (2 * s)][d][k] = P[k];
    __syncthreads();
    if ((c & (2 * s - 1)) == 0) { Dual Q[16], N[16]; for (int k = 0; k < 16; ++k) Q[k] = park[c / (2 * s)][d][k]; simu::mat4_mul(Q, P, N); for (int k = 0; k < 16; ++k) P[k] = N[k]; }
    __syncthreads();
  }
  if (c != 0) return;
  Dual r[3];
  simu::transition_residual(P, G.g01 + 6 * tr, G.g01 + 6 * tr + 3, r);
  double* o = G.out + (size_t)tr * kGyroOut;
  if (d == 0) for (int k = 0; k < 3; ++k) o[k] = r[k].v;
  if (d < G.np) for (int k = 0; k < 3; ++k) o[3 + 12 * k + d] = r[k].d;
}

// DataInterval::InitialInterval / TimeToIndex (imu_data_interval.h:104-118, :147-160): nearest-sample bisection, ties to the later index
int initial_interval_end(int n, const double* t, double duration) {
  const double end_ts = t[0] + duration;
  if (end_ts >= t[n - 1]) return n - 1;
  int i0 = 0, i1 = n - 1;
  while (i1 - i0 > 1) { const int im = (i0 + i1) / 2; if (end_ts > t[im]) i0 = im; else i1 = im; }
  return (end_ts - t[i0] < t[i1] - end_ts) ? i0 : i1;
}

void seq_mean(const double* x, int s, int e, double m[3]) {        // DataMean (imu_data_interval.cc:25-36)
  m[0] = m[1] = m[2] = 0.0;
  for (int i = s; i <= e; ++i) for (int d = 0; d < 3; ++d) m[d] += x[3 * (size_t)i + d];
  for (int d = 0; d < 3; ++d) m[d] /= (double)(e - s + 1);
}

}  // namespace

void default_static_imu_options(icc_static_imu_options* o) {
  memset(o, 0, sizeof *o);
  o->g_mag = 9.81; o->init_interval_duration_s = 30.0; o->gyro_dt = -1.0;
  o->interval_n_samples = 100; o->min_num_intervals = 12; o->win_size = 101;
  o->init_acc[3] = o->init_acc[4] = o->init_acc[5] = 1.0;
  o->init_gyr[6] = o->init_gyr[7] = o->init_gyr[8] = 1.0;
}

#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status static_imu_calibrate(cudaStream_t st, int n, const double* t, const double* acc, const double* gyr, const icc_static_imu_options& o,
                                double acc_out[9], double gyr_out[9], double bias_out[3], icc_static_imu_summary& S, std::vector<int32_t>& intervals, std::string& err) {
  const auto t_start = std::chrono::steady_clock::now();
  const int launches0 = kernel_launch_count();
  memset(&S, 0, sizeof S);
  intervals.clear();
  // the default (identity) triads: what getAccCalib / getGyroCalib return when the calibration fails (app :50-56)
  const double acc_id[9] = {0, 0, 0, 1, 1, 1, 0, 0, 0}, gyr_id[9] = {0, 0, 0, 0, 0, 0, 1, 1, 1};
  memcpy(acc_out, acc_id, sizeof acc_id); memcpy(gyr_out, gyr_id, sizeof gyr_id); bias_out[0] = bias_out[1] = bias_out[2] = 0.0;
  if (!(o.init_interval_duration_s > 0.0)) { err = "init_interval_duration_s must be positive"; return ICC_ERR_INVALID_ARGUMENT; }
  if (o.interval_n_samples < 1) { err = "interval_n_samples must be at least 1"; return ICC_ERR_INVALID_ARGUMENT; }
  for (int i = 1; i < n; ++i) if (!(t[i] >= t[i - 1])) { err = "timestamps must be non-decreasing"; return ICC_ERR_INVALID_ARGUMENT; }
  // ---- CalibrateAcc prologue (:63-79): initial interval statistics in the reference's sequential order -----------------------------
  const int e0 = initial_interval_end(n, t, o.init_interval_duration_s);
  double amean[3]; seq_mean(acc, 0, e0, amean);
  double var[3] = {0, 0, 0};
  for (int i = 0; i <= e0; ++i) for (int d = 0; d < 3; ++d) { const double df = acc[3 * (size_t)i + d] - amean[d]; var[d] += df * df; }
  for (int d = 0; d < 3; ++d) var[d] /= (double)(e0 + 1 - 1);
  const double norm_th = std::sqrt((var[0] * var[0] + var[1] * var[1]) + var[2] * var[2]);
  int imax = 0; for (int d = 1; d < 3; ++d) if (amean[d] > amean[imax]) imax = d;            // Eigen maxCoeff: first maximum, signed
  double x0[9] = {o.init_acc[0], o.init_acc[1], o.init_acc[2], o.init_acc[3], o.init_acc[4], o.init_acc[5], amean[0], amean[1], amean[2]};
  x0[6 + imax] -= o.g_mag;
  S.norm_threshold = norm_th;
  // ---- static detection, all ten multipliers ---------------------------------------------------------------------------------
  int win = o.win_size; if (win < 11) win = 11; if (!(win % 2)) win++;                        // :113-114
  const int h = win / 2;
  DevBuf<double> d_t, d_acc, d_gyr; CU(d_t.upload(t, n, st)); CU(d_acc.upload(acc, 3 * (size_t)n, st)); CU(d_gyr.upload(gyr, 3 * (size_t)n, st));
  std::vector<int> kept_n(kMult, 0);
  std::vector<std::vector<int2>> kept(kMult);
  if (win < n) {                                                                             // :118 (no intervals otherwise)
    const int nc = n - 2 * h, nb = (nc + kThreads - 1) / kThreads, cap = nc / 2 + 2;
    DevBuf<double> d_norm; CU(d_norm.alloc(n));
    const size_t smem = (size_t)(kThreads + 2 * h) * 3 * sizeof(double);
    const int stage = smem <= 48 * 1024 ? 1 : 0;
    window_norm_kernel<<<nb, kThreads, stage ? smem : 0, st>>>(n, h, d_acc.p, stage, d_norm.p); count_launch();
    DevBuf<int> d_counts, d_offsets, d_totals, d_starts, d_ends, d_ks, d_ke, d_kn;
    CU(d_counts.alloc(2 * kMult * (size_t)nb)); CU(d_offsets.alloc(2 * kMult * (size_t)nb)); CU(d_totals.alloc(2 * kMult));
    CU(d_starts.alloc(kMult * (size_t)cap)); CU(d_ends.alloc(kMult * (size_t)cap)); CU(d_ks.alloc(kMult * (size_t)cap)); CU(d_ke.alloc(kMult * (size_t)cap)); CU(d_kn.alloc(kMult));
    RunArgs R; R.n = n; R.h = h; R.nb = nb; R.cap = cap; R.norm = d_norm.p; R.counts = d_counts.p; R.offsets = d_offsets.p; R.starts = d_starts.p; R.ends = d_ends.p;
    for (int m = 0; m < kMult; ++m) R.thr[m] = (double)(m + 1) * norm_th;                       // th_mult * norm_th (:95)
    runs_kernel<<<nb, kThreads, 0, st>>>(R, 0); count_launch();
    block_scan_kernel<<<2 * kMult, kThreads, 0, st>>>(nb, d_counts.p, d_offsets.p, d_totals.p); count_launch();
    runs_kernel<<<nb, kThreads, 0, st>>>(R, 1); count_launch();
    keep_kernel<<<kMult, kThreads, 0, st>>>(cap, o.interval_n_samples, d_totals.p, d_starts.p, d_ends.p, d_ks.p, d_ke.p, d_kn.p); count_launch();
    CU(cudaMemcpyAsync(kept_n.data(), d_kn.p, kMult * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<int> ks, ke;
    for (int m = 0; m < kMult; ++m) {
      ks.resize(kept_n[m]); ke.resize(kept_n[m]);
      if (kept_n[m]) {
        CU(cudaMemcpyAsync(ks.data(), d_ks.p + (size_t)m * cap, kept_n[m] * sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(ke.data(), d_ke.p + (size_t)m * cap, kept_n[m] * sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
      }
      for (int k = 0; k < kept_n[m]; ++k) kept[m].push_back(make_int2(ks[k], ke[k]));
    }
  }
  for (int m = 0; m < kMult; ++m) {
    S.n_intervals[m] = kept_n[m];
    intervals.push_back(kept_n[m]);
    for (const int2& iv : kept[m]) { intervals.push_back(iv.x); intervals.push_back(iv.y); }
  }
  // ---- accelerometer fits, ten multipliers concurrently -----------------------------------------------------------------------
  AccFitArgs A; memset(&A, 0, sizeof A);
  std::vector<int2> all;
  bool any = false;
  for (int m = 0; m < kMult; ++m) {
    A.koff[m] = (int)all.size();
    all.insert(all.end(), kept[m].begin(), kept[m].end());
    A.fit[m] = kept_n[m] >= o.min_num_intervals ? 1 : 0;                                        // :106-110
    any = any || A.fit[m];
  }
  A.koff[kMult] = (int)all.size();
  int best = -1;
  std::vector<double> fit_out(kMult * kAccOut, 0.0);
  DevBuf<int2> d_all; DevBuf<double> d_means, d_fit;
  if (any) {
    CU(d_all.upload(all.data(), all.size(), st)); CU(d_means.alloc(3 * all.size())); CU(d_fit.alloc(fit_out.size()));
    if (o.acc_use_means) {
      AccTriad none; memset(&none, 0, sizeof none);
      interval_mean_kernel<<<((int)all.size() + 127) / 128, 128, 0, st>>>((int)all.size(), d_all.p, d_acc.p, 0, none, d_means.p); count_launch();
    }
    A.acc = d_acc.p; A.kept = d_all.p; A.means = d_means.p; A.ns = o.interval_n_samples; A.use_means = o.acc_use_means ? 1 : 0; A.g_mag = o.g_mag;
    memcpy(A.x0, x0, sizeof x0); A.o = ceres_default_options(); A.out = d_fit.p;
    acc_fit_kernel<<<kMult, kThreads, 0, st>>>(A); count_launch();
    CU(cudaMemcpyAsync(fit_out.data(), d_fit.p, fit_out.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    double min_cost = 1.7976931348623157e308;
    for (int m = 0; m < kMult; ++m) {
      if (!A.fit[m]) continue;
      const double* f = &fit_out[(size_t)m * kAccOut];
      for (int p = 0; p < 9; ++p) S.acc_params[m][p] = f[p];
      S.acc_initial_cost[m] = f[9]; S.acc_final_cost[m] = f[10]; S.acc_iterations[m] = (int)f[11]; S.acc_termination[m] = (int)f[12];
      if (f[10] < min_cost) { min_cost = f[10]; best = m; }                                      // strict < (:131-136)
    }
  }
  if (best < 0) {                                                                                // :140-146: CalibrateAccGyro returns false
    S.success = 0;
    S.gpu_launches = kernel_launch_count() - launches0;
    S.seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
    return ICC_OK;
  }
  S.chosen_multiplier = best + 1;
  for (int p = 0; p < 9; ++p) acc_out[p] = S.acc_params[best][p];
  // ---- CalibrateAccGyro (:188-337) ----------------------------------------------------------------------------------------------
  const int npos = kept_n[best];
  AccTriad tri;                                                                                  // ms = T K (types.h:318), bias
  {
    const double* q = acc_out;
    const double T[9] = {1.0, -q[0], q[1], 0.0, 1.0, -q[2], 0.0, 0.0, 1.0};
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) tri.ms[3 * r + c] = T[3 * r + c] * q[3 + c];
    for (int d = 0; d < 3; ++d) tri.b[d] = q[6 + d];
  }
  std::vector<double> gm(3 * (size_t)npos);
  interval_mean_kernel<<<(npos + 127) / 128, 128, 0, st>>>(npos, d_all.p + A.koff[best], d_acc.p, 1, tri, d_means.p); count_launch();
  CU(cudaMemcpyAsync(gm.data(), d_means.p, gm.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  double gbias[3]; seq_mean(gyr, 0, initial_interval_end(n, t, o.init_interval_duration_s), gbias);   // :214-218
  DevBuf<double> d_xg; CU(d_xg.alloc(3 * (size_t)n));
  unbias_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, d_gyr.p, gbias[0], gbias[1], gbias[2], d_xg.p); count_launch();
  CU(cudaStreamSynchronize(st));
  // transitions (:245-297): gravity directions and the monotone scan, here a bisection on the sorted timestamps
  const int ntr = npos - 1;
  std::vector<int2> span(std::max(ntr, 0));
  std::vector<double> g01(6 * (size_t)std::max(ntr, 0));
  int t_idx = 0;
  for (int i = 0; i < ntr; ++i) {
    for (int s = 0; s < 2; ++s) {
      const double* v = &gm[3 * (size_t)(i + s)];
      const double nv = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
      for (int d = 0; d < 3; ++d) g01[6 * (size_t)i + 3 * s + d] = v[d] / nv;
    }
    const double ts0 = t[kept[best][i].y], ts1 = t[kept[best][i + 1].x];
    const int i0 = (int)(std::lower_bound(t + t_idx, t + n, ts0) - t);
    int i1 = -1;
    if (i0 < n) {
      const int j = (int)(std::lower_bound(t + i0 + 1, t + n, ts1) - t);
      if (j < n) { i1 = j - 1; t_idx = j; } else t_idx = n;
    } else t_idx = n;
    span[i] = make_int2(i0 < n ? i0 : -1, i1);
    if (span[i].x < 0 || span[i].y < span[i].x) span[i] = make_int2(0, 0);                       // no samples: identity rotation
  }
  S.n_transitions = ntr;
  const int np = o.optimize_gyro_bias ? 12 : 9;
  double x[12];
  for (int p = 0; p < 9; ++p) x[p] = o.init_gyr[p];
  x[9] = x[10] = x[11] = 0.0;
  if (ntr > 0) {
    DevBuf<int2> d_span; DevBuf<double> d_g01, d_out;
    CU(d_span.upload(span.data(), ntr, st)); CU(d_g01.upload(g01.data(), g01.size(), st)); CU(d_out.alloc(kGyroOut * (size_t)ntr));
    CU(cudaMemsetAsync(d_out.p, 0, kGyroOut * (size_t)ntr * sizeof(double), st));
    GyroArgs G; memset(&G, 0, sizeof G);
    G.x = d_xg.p; G.t = d_t.p; G.span = d_span.p; G.g01 = d_g01.p; G.gyro_dt = o.gyro_dt; G.np = np; G.with_bias = o.optimize_gyro_bias ? 1 : 0; G.out = d_out.p;
    std::vector<double> out(kGyroOut * (size_t)ntr);
    double H[12][12], g[12], cost;
    auto eval = [&](const double* xp) -> icc_status {
      for (int p = 0; p < 12; ++p) G.p[p] = xp[p];
      gyro_eval_kernel<<<ntr, kChunks * kDirs, 0, st>>>(G); count_launch();
      CU(cudaMemcpyAsync(out.data(), d_out.p, out.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      CU(cudaGetLastError());
      for (int p = 0; p < 12; ++p) { g[p] = 0.0; for (int q = 0; q < 12; ++q) H[p][q] = 0.0; }
      double c2 = 0.0;
      for (int i = 0; i < ntr; ++i) {
        const double* o_ = &out[(size_t)i * kGyroOut];
        for (int k = 0; k < 3; ++k) {
          const double r = o_[k], *J = o_ + 3 + 12 * k;
          c2 += r * r;
          for (int p = 0; p < np; ++p) { g[p] += J[p] * r; for (int q = 0; q < np; ++q) H[p][q] += J[p] * J[q]; }
        }
      }
      cost = 0.5 * c2;
      return ICC_OK;
    };
    icc_status rc = eval(x); if (rc != ICC_OK) return rc;
    LmState L;
    simu::lm_start(L, ceres_default_options(), np, x, cost, H, g);
    while (simu::lm_propose(L)) {
      rc = eval(L.xc); if (rc != ICC_OK) return rc;
      simu::lm_consider(L, cost, H, g);
    }
    for (int p = 0; p < 12; ++p) x[p] = L.x[p];
    S.gyro_initial_cost = L.T.initial_cost; S.gyro_final_cost = L.T.cost; S.gyro_iterations = L.T.iterations; S.gyro_termination = L.T.termination;
  }
  for (int p = 0; p < 9; ++p) gyr_out[p] = x[p];
  for (int d = 0; d < 3; ++d) bias_out[d] = gbias[d] + x[9 + d];                                  // :320-331
  S.success = 1;
  S.gpu_launches = kernel_launch_count() - launches0;
  S.seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
  return ICC_OK;
}

}  // namespace icc
