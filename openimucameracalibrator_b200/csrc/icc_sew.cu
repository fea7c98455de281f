// Spline Error Weighting (sm_90a): knot spacing + spline-fit variance from the spectrum of an IMU stream, i.e. the
// `spline_error_weighting_json` the hot CLI requires (SURVEY.md §8(f) row f2).
//
// Replaces python/sew.py:knot_spacing_and_variance (python/sew.py:86-147,150-234) as driven by python/get_sew_for_dataset.py:38-48:
//   Xhat[k] = sqrt(1/d) * || FFT(signal)[:, k] ||  with the DC bin removed                     (make_reference_spectrum, :171-181)
//   quality(dt) = (1 - q) * E(Xhat) / E((1 - H(f; dt)) * Xhat),  E(X) = sum |X|^2 / N          (:148-154, signal_energy :82-83)
//   H(f; dt) = 3 sinc(f dt)^4 / (2 + cos(2 pi f dt))    cubic B-spline interpolation response  (:36-80)
//   dt = largest spacing in [min_dt, max_dt] with quality >= 1: end-point test, halving back-track, Brent root (:86-145)
//   variance = E((1 - H(f; dt)) * Xhat) / N                                                      (:196-199)
//
// Mapping to the machine: the length-N DFT (N arbitrary: 100 k samples for BASELINE config 4) is Bluestein's chirp-z transform on
// power-of-two Stockham radix-2 passes written here (FP64, twiddles from sincospi, chirp phase reduced with exact integer
// arithmetic n^2 mod 2N), batched over the three axes; the spectrum stays in HBM and each quality evaluation of the root search
// is one fused response + energy reduction over the N bins.  The scalar root search (a dozen evaluations) runs on the host.
#include "icc_kernels.h"

#include <cmath>

namespace icc {

void count_launch();

namespace {

struct cplx { double re, im; };
__device__ __forceinline__ cplx cmul(cplx a, cplx b) { return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }

// chirp w_n = exp(-i pi n^2 / N); the phase is reduced exactly: n^2 mod 2N
__device__ __forceinline__ cplx chirp(long long n, long long N) {
  const long long r = (n * n) % (2 * N);
  double s, c; sincospi(-(double)r / (double)N, &s, &c);
  return {c, s};
}

// a[ch][m] = x[ch][m] w_m (m < N), 0 beyond ; b[m] = conj(w_m) for |m| < N wrapped into [0, M)
__global__ void bluestein_setup_kernel(int N, int M, const double* __restrict__ x /* N x 3 */, cplx* __restrict__ a /* 3 x M */, cplx* __restrict__ b /* M */) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  cplx w = {0.0, 0.0};
  if (m < N) w = chirp(m, N);
  for (int ch = 0; ch < 3; ++ch) { cplx v = {0.0, 0.0}; if (m < N) { const double s = x[3 * (size_t)m + ch]; v = {s * w.re, s * w.im}; } a[(size_t)ch * M + m] = v; }
  cplx bv = {0.0, 0.0};
  if (m < N) bv = {w.re, -w.im};
  else if (m > M - N) { const cplx wm = chirp(M - m, N); bv = {wm.re, -wm.im}; }
  b[m] = bv;
}

// one Stockham radix-2 pass over `batch` transforms of length M (autosort: no bit reversal); sign = -1 forward, +1 inverse
// in -> out, half = M / 2, stride `s` = 1, 2, 4, ... ; butterfly j in [0, half): p = j / s, q = j % s
__global__ void stockham_pass_kernel(int M, int s, int sign, const cplx* __restrict__ in, cplx* __restrict__ out) {
  const int half = M >> 1;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= half) return;
  const cplx* src = in + (size_t)blockIdx.y * M; cplx* dst = out + (size_t)blockIdx.y * M;
  const int q = j & (s - 1), p = j / s;            // s is a power of two
  // n = M / s current sub-transform length: twiddle exp(sign * 2 pi i p / n) = exp(sign * 2 pi i (p s) / M)
  double sn, cs; sincospi((double)sign * 2.0 * (double)((long long)p * s) / (double)M, &sn, &cs);
  const cplx a = src[q + s * p], b = src[q + s * (p + half / s)];
  const cplx d = {a.re - b.re, a.im - b.im};
  dst[q + s * (2 * p)] = {a.re + b.re, a.im + b.im};
  dst[q + s * (2 * p + 1)] = cmul(d, cplx{cs, sn});
}

__global__ void pointwise_mul_kernel(int M, cplx* __restrict__ A /* 3 x M */, const cplx* __restrict__ B /* M */) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const cplx bv = B[m];
  for (int ch = 0; ch < 3; ++ch) A[(size_t)ch * M + m] = cmul(A[(size_t)ch * M + m], bv);
}

// X_k = w_k c_k / M (inverse transform scaling) ; Xhat_k = sqrt(1/3 sum_ch |X_ch,k|^2), Xhat_0 = 0 ; energy += Xhat_k^2
__global__ void spectrum_kernel(int N, int M, const cplx* __restrict__ c /* 3 x M */, double* __restrict__ xhat, double* __restrict__ energy_sum) {
  __shared__ double red[8];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  double e = 0.0;
  if (k < N) {
    const cplx w = chirp(k, N);
    double s2 = 0.0;
    for (int ch = 0; ch < 3; ++ch) { const cplx v = cmul(c[(size_t)ch * M + k], w); const double re = v.re / M, im = v.im / M; s2 += re * re + im * im; }
    const double xh = k == 0 ? 0.0 : sqrt(1.0 / 3.0) * sqrt(s2);
    xhat[k] = xh; e = xh * xh;
  }
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0.0; for (int w2 = 0; w2 < (blockDim.x >> 5); ++w2) t += red[w2]; atomicAdd(energy_sum, t); }
}

// sum_k ((1 - H(f_k; dt)) Xhat_k)^2 with f_k = fftfreq(N, d)[k] = i_k * fscale
__global__ void residual_energy_kernel(int N, const double* __restrict__ xhat, double fscale, double dt, double* __restrict__ out) {
  __shared__ double red[8];
  double e = 0.0;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < N; k += gridDim.x * blockDim.x) {
    const int ik = k < (N + 1) / 2 ? k : k - N;
    const double y = (double)ik * fscale * dt;       // f dt
    double sinc = 1.0;
    if (y != 0.0) { const double py = 3.14159265358979323846 * y; sinc = sin(py) / py; }
    const double s2 = sinc * sinc, H = 3.0 * s2 * s2 / (2.0 + cos(2.0 * 3.14159265358979323846 * y));
    const double v = (1.0 - H) * xhat[k];
    e += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0.0; for (int w2 = 0; w2 < (blockDim.x >> 5); ++w2) t += red[w2]; atomicAdd(out, t); }
}

}  // namespace

int sew_fft_length(int N) { int M = 1; while (M < 2 * N - 1) M <<= 1; return M; }

// xhat[N] <- reference spectrum of signal (N x 3) ; *energy_sum <- sum xhat^2 ; scratch: 2 x (3 M + M) complex = 16 M doubles
void launch_sew_spectrum(int N, const double* signal, double* xhat, double* energy_sum, double* scratch, cudaStream_t st) {
  const int M = sew_fft_length(N);
  cplx* bufA = reinterpret_cast<cplx*>(scratch);            // 4 x M: [a0 a1 a2 | b]
  cplx* bufB = bufA + (size_t)4 * M;                        // ping-pong partner
  bluestein_setup_kernel<<<(M + 255) / 256, 256, 0, st>>>(N, M, signal, bufA, bufA + (size_t)3 * M); count_launch();
  cplx* src = bufA; cplx* dst = bufB;
  const dim3 grid((M / 2 + 255) / 256, 4);
  for (int s = 1; s < M; s <<= 1) { stockham_pass_kernel<<<grid, 256, 0, st>>>(M, s, -1, src, dst); count_launch(); cplx* t = src; src = dst; dst = t; }
  pointwise_mul_kernel<<<(M + 255) / 256, 256, 0, st>>>(M, src, src + (size_t)3 * M); count_launch();
  const dim3 grid3((M / 2 + 255) / 256, 3);
  for (int s = 1; s < M; s <<= 1) { stockham_pass_kernel<<<grid3, 256, 0, st>>>(M, s, +1, src, dst); count_launch(); cplx* t = src; src = dst; dst = t; }
  cudaMemsetAsync(energy_sum, 0, sizeof(double), st);
  spectrum_kernel<<<(N + 255) / 256, 256, 0, st>>>(N, M, src, xhat, energy_sum); count_launch();
}

void launch_sew_residual_energy(int N, const double* xhat, double fscale, double dt, double* out, int sm_count, cudaStream_t st) {
  cudaMemsetAsync(out, 0, sizeof(double), st);
  int g = (N + 255) / 256; if (g > 4 * sm_count) g = 4 * sm_count; if (g < 1) g = 1;
  residual_energy_kernel<<<g, 256, 0, st>>>(N, xhat, fscale, dt, out); count_launch();
}

// ---- static IMU biases (python/get_imu_biases.py:36-53): column sums of the accelerometer and gyroscope streams -------------------
namespace {
__global__ void __launch_bounds__(256) imu_sums_kernel(int n, const double* __restrict__ acc, const double* __restrict__ gyr, double* __restrict__ out /* 6 */) {
  double s[6] = {0, 0, 0, 0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    s[0] += acc[3 * i]; s[1] += acc[3 * i + 1]; s[2] += acc[3 * i + 2]; s[3] += gyr[3 * i]; s[4] += gyr[3 * i + 1]; s[5] += gyr[3 * i + 2];
  }
  __shared__ double sh[8][6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double v = s[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sh[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) { double v = 0.0; for (int w = 0; w < 8; ++w) v += sh[w][threadIdx.x]; atomicAdd(&out[threadIdx.x], v); }
}
}  // namespace

void launch_imu_sums(int n, const double* acc, const double* gyr, double* out6, int sm_count, cudaStream_t st) {
  cudaMemsetAsync(out6, 0, 6 * sizeof(double), st);
  if (n <= 0) return;
  int g = (n + 255) / 256; if (g > 4 * sm_count) g = 4 * sm_count;
  imu_sums_kernel<<<g, 256, 0, st>>>(n, acc, gyr, out6); count_launch();
}

}  // namespace icc

