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
#include "icc_host.h"
#include "icc_reduce.cuh"

#include <cmath>
#include <functional>

namespace icc {

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
  e = warp_sum(e);   // one sum: thread 0 adds the warps in order behind a single barrier, where block_sums<1> would take two
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
  e = warp_sum(e);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0.0; for (int w2 = 0; w2 < (blockDim.x >> 5); ++w2) t += red[w2]; atomicAdd(out, t); }
}

// scipy.optimize.brentq (Brent 1973 as implemented in scipy/optimize/Zeros/brentq.c), xtol = 2e-12, rtol = 4 eps, 100 iterations
double brentq(const std::function<double(double)>& f, double xa, double xb, bool& ok) {
  const double xtol = 2e-12, rtol = 8.881784197001252e-16;
  double xpre = xa, xcur = xb, xblk = 0.0, fpre = f(xpre), fcur = f(xcur), fblk = 0.0, spre = 0.0, scur = 0.0;
  ok = true;
  if (fpre == 0.0) return xpre;
  if (fcur == 0.0) return xcur;
  if ((fpre > 0) == (fcur > 0)) { ok = false; return xcur; }
  for (int i = 0; i < 100; ++i) {
    if (fpre != 0.0 && fcur != 0.0 && ((fpre > 0) != (fcur > 0))) { xblk = xpre; fblk = fpre; spre = scur = xcur - xpre; }
    if (std::fabs(fblk) < std::fabs(fcur)) { xpre = xcur; xcur = xblk; xblk = xpre; fpre = fcur; fcur = fblk; fblk = fpre; }
    const double delta = (xtol + rtol * std::fabs(xcur)) / 2, sbis = (xblk - xcur) / 2;
    if (fcur == 0.0 || std::fabs(sbis) < delta) return xcur;
    if (std::fabs(spre) > delta && std::fabs(fcur) < std::fabs(fpre)) {
      double stry;
      if (xpre == xblk) stry = -fcur * (xcur - xpre) / (fcur - fpre);                       // secant
      else { const double dpre = (fpre - fcur) / (xpre - xcur), dblk = (fblk - fcur) / (xblk - xcur); stry = -fcur * (fblk * dblk - fpre * dpre) / (dblk * dpre * (fblk - fpre)); }   // inverse quadratic
      if (2 * std::fabs(stry) < std::min(std::fabs(spre), 3 * std::fabs(sbis) - delta)) { spre = scur; scur = stry; }
      else { spre = sbis; scur = sbis; }
    } else { spre = sbis; scur = sbis; }
    xpre = xcur; fpre = fcur;
    if (std::fabs(scur) > delta) xcur += scur; else xcur += (sbis > 0 ? delta : -delta);
    fcur = f(xcur);
  }
  ok = false;
  return xcur;
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
  __shared__ double red[8][6], tot[6];
  block_sums<6>(s, red, tot);
  if (threadIdx.x < 6) atomicAdd(&out[threadIdx.x], tot[threadIdx.x]);
}
}  // namespace

void launch_imu_sums(int n, const double* acc, const double* gyr, double* out6, int sm_count, cudaStream_t st) {
  cudaMemsetAsync(out6, 0, 6 * sizeof(double), st);
  if (n <= 0) return;
  int g = (n + 255) / 256; if (g > 4 * sm_count) g = 4 * sm_count;
  imu_sums_kernel<<<g, 256, 0, st>>>(n, acc, gyr, out6); count_launch();
}

// ---- host drivers: row f2 (icc_spline_error_weighting) and the static IMU biases (icc_estimate_imu_biases) -----------------------
#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status spline_error_weighting(cudaStream_t st, int sm_count, int n, const double* times, const double* signal, double quality, double min_dt, double max_dt, double* dt_out, double* var_out, double* spectrum, std::string& err) {
  double mean_dt = 0.0; for (int i = 1; i < n; ++i) mean_dt += times[i] - times[i - 1]; mean_dt /= (double)(n - 1);
  if (!(mean_dt > 0.0)) { err = "timestamps must increase on average"; return ICC_ERR_INVALID_ARGUMENT; }
  const double sample_rate = 1.0 / mean_dt, d = 1.0 / sample_rate, fscale = 1.0 / ((double)n * d);   // np.fft.fftfreq(n, d): k * (1 / (n d))
  if (!(min_dt > 0.0)) min_dt = 1.0 / sample_rate;                                                     // sew.py:156-160
  if (!(max_dt > 0.0)) max_dt = ((double)n / 4.0) / sample_rate;
  const int M = sew_fft_length(n);
  DevBuf<double> d_sig, d_xhat, d_scr, d_acc;
  CU(d_sig.upload(signal, 3 * (size_t)n, st)); CU(d_xhat.alloc(n)); CU(d_scr.alloc(16 * (size_t)M)); CU(d_acc.alloc(2));
  launch_sew_spectrum(n, d_sig.p, d_xhat.p, d_acc.p, d_scr.p, st);
  double esum = 0.0;
  CU(cudaMemcpyAsync(&esum, d_acc.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  if (spectrum) CU(cudaMemcpyAsync(spectrum, d_xhat.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (cudaGetLastError() != cudaSuccess) { err = "spectrum kernels failed"; return ICC_ERR_CUDA; }
  const double max_remove = esum / (double)n * (1.0 - quality);                                        // signal_energy(Xhat) * (1 - quality)
  bool cuda_ok = true;
  auto removed = [&](double dt) -> double {      // signal_energy((1 - H) * Xhat)
    double e = 0.0;
    launch_sew_residual_energy(n, d_xhat.p, fscale, dt, d_acc.p + 1, sm_count > 0 ? sm_count : 132, st);
    if (cudaMemcpyAsync(&e, d_acc.p + 1, sizeof(double), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) cuda_ok = false;
    return e / (double)n;
  };
  auto quality_func = [&](double dt) { return max_remove / removed(dt); };
  // find_max_quality_dt(quality_func, 1.0, min_dt, max_dt)   (sew.py:86-145)
  double dt = max_dt, found = 0.0; bool have = false;
  if (quality_func(dt) >= 1.0) { found = dt; have = true; }
  else {
    double step = max_dt * 0.5, max_quality = 0.0, max_quality_dt = dt; bool any = false;
    while (!have) {
      dt -= step; dt = std::max(dt, min_dt);
      const double q = quality_func(dt);
      if (q > 1.0) { bool ok; found = brentq([&](double x) { return quality_func(x) - 1.0; }, dt, max_dt, ok); if (!ok) { err = "Brent root search failed"; return ICC_ERR_NUMERIC; } have = true; }
      else {
        step *= 0.5;
        if (q > max_quality) { max_quality = q; max_quality_dt = dt; any = true; }
        if (dt <= min_dt) { if (!any) { err = "no knot spacing satisfies the quality"; return ICC_ERR_NUMERIC; } found = max_quality_dt; have = true; }
      }
      if (!cuda_ok) { err = "quality kernels failed"; return ICC_ERR_CUDA; }
    }
  }
  *dt_out = found;
  *var_out = removed(found) / (double)n;                                                               // dt_to_variance_spectrum (:196-199)
  if (!cuda_ok) { err = "quality kernels failed"; return ICC_ERR_CUDA; }
  return ICC_OK;
}

// python/get_imu_biases.py:36-53
icc_status imu_biases(cudaStream_t st, int sm_count, int n, const double* acc, const double* gyr, double gravity_const, double accl_bias[3], double gyro_bias[3], std::string& err) {
  DevBuf<double> d_a, d_g, d_s;
  CU(d_a.upload(acc, 3 * (size_t)n, st)); CU(d_g.upload(gyr, 3 * (size_t)n, st)); CU(d_s.alloc(6));
  launch_imu_sums(n, d_a.p, d_g.p, d_s.p, sm_count, st);
  double s[6];
  CU(cudaMemcpyAsync(s, d_s.p, sizeof s, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (cudaGetLastError() != cudaSuccess) { err = "bias kernel failed"; return ICC_ERR_CUDA; }
  double mean_a[3], mean_g[3];
  for (int d = 0; d < 3; ++d) { mean_a[d] = s[d] / n; mean_g[d] = s[3 + d] / n; }
  int ax = 0; for (int d = 1; d < 3; ++d) if (std::fabs(mean_a[d]) > std::fabs(mean_a[ax])) ax = d;          // :39-41 (first maximum)
  const double sgn = mean_a[ax] > 0.0 ? 1.0 : (mean_a[ax] < 0.0 ? -1.0 : 0.0);
  const double grav = (double)(float)(gravity_const * sgn);                                                     // float32 array (:43-44)
  for (int d = 0; d < 3; ++d) { accl_bias[d] = mean_a[d] - (d == ax ? grav : 0.0); gyro_bias[d] = mean_g[d]; }   // :46, :49-50
  return ICC_OK;
}

}  // namespace icc

