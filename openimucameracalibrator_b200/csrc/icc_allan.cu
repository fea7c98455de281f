// Allan variance noise characterisation of a static IMU log (sm_90a): what the reference's fit_allan_variance tool computes.
//
// Replaces what the reference runs serially on the CPU in
//   AllanVarianceFitter::RunFit                          src/core/allan_variance_fitter.cc
//   AllanGyr / AllanAcc::calc, calcVariance, ...          src/allanvariance/allan_gyr.cc, allan_acc.cc
//   FitAllanGyr / FitAllanAcc (ceres::Solve, DOGLEG)       src/allanvariance/fitallan_gyr.cc, fitallan_acc.cc
// The reference computes, per channel, an overlapping Allan variance at F (about 6000) cluster sizes m: F sums of n - 2m squared
// second differences of the integrated signal, about 10^4 n terms, and RunFit computes every curve twice.  Here:
//   * the integrated signal theta = cumsum(x) / freq is the reference's sequential running sum, one warp per channel, so theta is
//     bit for bit the reference's (a blocked parallel scan rounds differently, which moves sigma^2 by up to ~2e-9 relative on a
//     channel dominated by a constant such as gravity);
//   * one launch computes every sigma^2(m) of every channel once.  A CTA owns (k slice, group of up to 16 consecutive factors whose
//     span is at most kSpan, channel).  Per tile of kTile k-values it stages theta[k0, k0 + kTile), theta[k0 + m_first, k0 + m_last +
//     kTile) and theta[k0 + 2 m_first, k0 + 2 m_last + kTile) in shared memory, and each warp sums its two factors of the group from
//     those windows (the first window is read once for both).  A lane keeps its sums in registers across the slice's tiles; the
//     warp reduces them with shuffles and writes one partial per (channel, factor, slice).  A second kernel adds the partials of a
//     factor in slice order and divides by the reference's divisor: deterministic, no atomics;
//   * the six fits run concurrently, one CTA each, the whole dogleg loop inside the kernel (closed-form Jacobian rows, block-reduced
//     5x5 normal equations, one-thread step control in icc_allan_math.cuh / icc_trust_region.cuh).
//   The factor set, the accelerometer point filter and the initial values (a 5x5 least-squares problem) are host code.
#include "../../include/icc_b200.h"
#include "icc_allan_math.cuh"
#include "icc_host.h"
#include "icc_reduce.cuh"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace icc {

namespace {

constexpr int kThreads = 256;
constexpr int kThetaChunk = 2048;                              // samples staged per step of the running sum
constexpr int kTile = 2048, kSpan = 1024, kGroup = 16;         // variance: k-values per tile, factor span and count per group
constexpr int kTilesPerSlice = 8, kSlice = kTile * kTilesPerSlice;
constexpr int kGroupGrid = 1024;                               // grid.y: groups beyond it are a grid-stride loop
constexpr int kSmemDoubles = 3 * kTile + 3 * kSpan;
constexpr int kFitSums = normal_equation_sums(5);
constexpr int kFitOut = 10;                                    // x[5], initial cost, final cost, iterations, termination, successful

// the sample of channel c (0-2 accelerometer x, y, z as given; 3-5 gyroscope x, y, z pushed as rad/s, i.e. x * 57.3 * 3600)
ICC_D double sample(const double* __restrict__ acc, const double* __restrict__ gyr, int c, size_t k) {
  return c < 3 ? acc[3 * k + c] : __dmul_rn(__dmul_rn(gyr[3 * k + c - 3], 57.3), 3600.0);   // not contracted into the running sum
}

// theta[c][k] = (sum of the samples 0..k) / freq, the reference's sequential running sum (calcThetas) bit for bit, and total[c] =
// the channel's sum (getAvgValue's).  One warp per channel: the lanes stage a chunk in shared memory, lane 0 adds it up in order.
__global__ void theta_kernel(int n, double freq, const double* __restrict__ acc, const double* __restrict__ gyr, double* __restrict__ theta,
                             double* __restrict__ total) {
  __shared__ double buf[kThetaChunk];
  const int c = blockIdx.x, lane = threadIdx.x;
  double* th = theta + (size_t)c * n;
  double s = 0.0;
  for (int base = 0; base < n; base += kThetaChunk) {
    const int len = min(kThetaChunk, n - base);
    for (int i = lane; i < len; i += 32) buf[i] = sample(acc, gyr, c, (size_t)base + i);
    __syncwarp();
    if (lane == 0)
#pragma unroll 8
      for (int i = 0; i < len; ++i) { s += buf[i]; buf[i] = s; }
    __syncwarp();
    for (int i = lane; i < len; i += 32) th[base + i] = buf[i] / freq;
    __syncwarp();
  }
  if (lane == 0) total[c] = s;
}

struct VarArgs {
  const double* theta;     // 6 x n
  const int* m;            // factors (F)
  const int* gfirst;       // per group: first factor index, factor count
  const int* gcount;
  double* partial;         // 6 x F x nslice
  int n, F, G, nslice;
};

// sum over k in the CTA's slice of (theta[k + 2m] - 2 theta[k + m] + theta[k])^2 for the group's factors (calcVariance's inner loop).
// The groups are a grid-stride loop over grid.y (kGroupGrid, one group per CTA at the default 10000 clusters), so any n_clusters
// launches within grid.y's limit of 65535.
__global__ void __launch_bounds__(kThreads) variance_kernel(VarArgs A) {
  extern __shared__ double sm[];
  const int s = blockIdx.x, c = blockIdx.z, n = A.n;
  const int kbeg = s * kSlice;
  const double* __restrict__ th = A.theta + (size_t)c * n;
  double* W0 = sm;
  double* W1 = W0 + kTile;
  double* W2 = W1 + kTile + kSpan;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int g = blockIdx.y; g < A.G; g += gridDim.y) {
    const int f0 = A.gfirst[g], nf = A.gcount[g];
    const int ma = A.m[f0], mb = A.m[f0 + nf - 1];
    const int kend = n - 2 * ma;
    if (kbeg >= kend) continue;   // block-uniform
    const int L1 = kTile + (mb - ma), L2 = kTile + 2 * (mb - ma);
    const bool has1 = warp < nf, has2 = warp + 8 < nf;
    const int m1 = has1 ? A.m[f0 + warp] : ma, m2 = has2 ? A.m[f0 + warp + 8] : ma;
    const int e1 = has1 ? n - 2 * m1 : 0, e2 = has2 ? n - 2 * m2 : 0;   // k < e: the factor's terms
    const int d1 = m1 - ma, d2 = m2 - ma;
    double acc1 = 0.0, acc2 = 0.0;
    for (int t = 0; t < kTilesPerSlice; ++t) {
      const int k0 = kbeg + t * kTile;
      if (k0 >= kend) break;
      __syncthreads();   // the previous tile (or group) is consumed
      for (int i = threadIdx.x; i < kTile; i += kThreads) W0[i] = k0 + i < n ? th[k0 + i] : 0.0;
      for (int i = threadIdx.x; i < L1; i += kThreads) { const int k = k0 + ma + i; W1[i] = k < n ? th[k] : 0.0; }
      for (int i = threadIdx.x; i < L2; i += kThreads) { const int k = k0 + 2 * ma + i; W2[i] = k < n ? th[k] : 0.0; }
      __syncthreads();
      if (!has1) continue;
      for (int i = lane; i < kTile; i += 32) {
        const int k = k0 + i;
        if (k >= e1) break;   // e2 <= e1
        const double a0 = W0[i];
        const double u = (W2[i + 2 * d1] - 2 * W1[i + d1]) + a0;
        acc1 += u * u;
        if (k < e2) { const double w = (W2[i + 2 * d2] - 2 * W1[i + d2]) + a0; acc2 += w * w; }
      }
    }
    acc1 = warp_sum(acc1); acc2 = warp_sum(acc2);
    if (lane == 0) {
      if (has1) A.partial[((size_t)c * A.F + f0 + warp) * A.nslice + s] = acc1;
      if (has2) A.partial[((size_t)c * A.F + f0 + warp + 8) * A.nslice + s] = acc2;
    }
  }
}

// sigma2 = (partials of the factor's slices, in order) / 2 (period m)^2 (n - 2m)
__global__ void variance_finish_kernel(int n, int F, int nslice, const int* __restrict__ m, const double* __restrict__ div,
                                       const double* __restrict__ partial, double* __restrict__ sigma2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 6 * F) return;
  const int f = i % F;
  const int terms = n - 2 * m[f];
  const int ns = terms > 0 ? (terms + kSlice - 1) / kSlice : 0;
  double s = 0.0;
  for (int q = 0; q < ns; ++q) s += partial[(size_t)i * nslice + q];
  sigma2[i] = s / div[f];
}

struct FitArgs {
  const double* tau;       // fit points of all channels, concatenated
  const double* l10s;      // log10(sigma2) of the points
  int off[7];              // channel c: points [off[c], off[c+1])
  double x0[6][5];
  double* out;             // per channel kFitOut values
};

// cost, J^T J, J^T r of channel c's points at x, reduced over the block in a fixed order; valid in every thread after the call
ICC_D void fit_normal_equations(const FitArgs& A, int c, const double* x, double (*red)[kFitSums], double* tot) {
  double s[kFitSums];
#pragma unroll
  for (int k = 0; k < kFitSums; ++k) s[k] = 0.0;
  for (int j = A.off[c] + threadIdx.x; j < A.off[c + 1]; j += blockDim.x) {
    double J[5];
    const double r = allan::residual(x, A.tau[j], A.l10s[j], J);
    normal_equation_row<5>(s, J, r);
  }
  block_sums<kFitSums>(s, red, tot);
}

// one CTA per channel: the reference's ceres::Solve (fitallan_gyr.cc:21-40) entirely on the device.  Thread 0 owns the minimiser
// state; the block evaluates the normal equations at the point thread 0 publishes in x.
__global__ void __launch_bounds__(kThreads) fit_kernel(FitArgs A) {
  __shared__ double red[kThreads / 32][kFitSums];
  __shared__ double tot[kFitSums];
  __shared__ double x[5];
  __shared__ int go;
  const int c = blockIdx.x;
  allan::Fit F;
  if (threadIdx.x < 5) x[threadIdx.x] = A.x0[c][threadIdx.x];
  __syncthreads();
  fit_normal_equations(A, c, x, red, tot);
  if (threadIdx.x == 0) { double H[5][5], b[5], cost; unpack_normal_equations<5, 5>(tot, H, b, cost); allan::fit_start(F, A.x0[c], cost, H, b); }
  for (;;) {
    if (threadIdx.x == 0) { go = allan::fit_propose(F) ? 1 : 0; for (int p = 0; p < 5; ++p) x[p] = F.xc[p]; }
    __syncthreads();
    if (!go) break;
    fit_normal_equations(A, c, x, red, tot);
    if (threadIdx.x == 0) { double H[5][5], b[5], cost; unpack_normal_equations<5, 5>(tot, H, b, cost); allan::fit_consider(F, cost, H, b); }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* o = A.out + (size_t)c * kFitOut;
    for (int p = 0; p < 5; ++p) o[p] = F.x[p];
    o[5] = F.D.T.initial_cost; o[6] = F.D.T.cost; o[7] = F.D.T.iterations; o[8] = F.D.T.termination; o[9] = F.D.T.successful;
  }
}

// findMinNum / findMinIndex (fitallan_gyr.cc:123-138): both start from 1000, ties go to the later index
void min_deviation(const double p[5], const std::vector<double>& tau, double& dmin, int& imin) {
  dmin = 1000.0; imin = 0;
  for (size_t i = 0; i < tau.size(); ++i) {
    const double d = std::sqrt(allan::model(p, tau[i]));
    imin = dmin < d ? imin : (int)i;
    dmin = dmin < d ? dmin : d;
  }
}

}  // namespace

void default_allan_options(icc_allan_options* o) {
  memset(o, 0, sizeof *o);
  o->n_clusters = 10000;   // AllanVarianceFitter(telemetry, 10000) (applications/fit_allan_variance.cc:41)
}

#define CU(call) ICC_CUDA_CHECK(call, err)

icc_status allan_variance(cudaStream_t st, int n, const double* t, const double* acc, const double* gyr, const icc_allan_options& o,
                          double params[30], icc_allan_noise noise[6], icc_allan_summary summary[6], allan::Curves& curves, std::string& err) {
  const auto t_start = std::chrono::steady_clock::now();
  const int launches0 = kernel_launch_count();
  if (n < 3) { err = "need at least 3 samples"; return ICC_ERR_INVALID_ARGUMENT; }
  if (o.n_clusters < 2) { err = "n_clusters must be at least 2"; return ICC_ERR_INVALID_ARGUMENT; }
  // getAvgDt (allan_gyr.cc:199-209): mean of the consecutive differences; freq = 1 / dt, period = dt
  double sum_dt = 0.0;
  for (int i = 1; i < n; ++i) sum_dt += t[i] - t[i - 1];
  const double period = sum_dt / (n - 1), freq = 1.0 / period;
  // ---- factors, groups, divisors (host) ---------------------------------------------------------------------------------------
  const std::vector<int> m = allan::factors(n, o.n_clusters);
  const int F = (int)m.size();
  std::vector<int> gfirst, gcount;
  for (int f = 0; f < F;) {
    int e = f + 1;
    while (e < F && e - f < kGroup && m[e] - m[f] <= kSpan) ++e;
    gfirst.push_back(f); gcount.push_back(e - f); f = e;
  }
  const int G = (int)gfirst.size();
  std::vector<double> div(F);
  curves.factors = m; curves.tau.assign(F, 0.0);
  for (int f = 0; f < F; ++f) { div[f] = allan::variance_divisor(period, m[f], n); curves.tau[f] = period * m[f]; }   // getTimes
  const int nslice = std::max(1, (n + kSlice - 1) / kSlice);
  // ---- theta and the variance of all six channels --------------------------------------------------------------------------------
  DevBuf<double> d_acc, d_gyr, d_total, d_theta, d_partial, d_div, d_sigma2;
  DevBuf<int> d_m, d_gfirst, d_gcount;
  CU(d_acc.upload(acc, 3 * (size_t)n, st)); CU(d_gyr.upload(gyr, 3 * (size_t)n, st)); CU(d_m.upload(m.data(), F, st));
  CU(d_gfirst.upload(gfirst.data(), G, st)); CU(d_gcount.upload(gcount.data(), G, st)); CU(d_div.upload(div.data(), F, st));
  CU(d_total.alloc(6)); CU(d_theta.alloc(6 * (size_t)n)); CU(d_partial.alloc(6 * (size_t)F * nslice)); CU(d_sigma2.alloc(6 * (size_t)F));
  theta_kernel<<<6, 32, 0, st>>>(n, freq, d_acc.p, d_gyr.p, d_theta.p, d_total.p); count_launch();
  VarArgs V; V.theta = d_theta.p; V.m = d_m.p; V.gfirst = d_gfirst.p; V.gcount = d_gcount.p; V.partial = d_partial.p; V.n = n; V.F = F; V.G = G; V.nslice = nslice;
  const size_t smem = kSmemDoubles * sizeof(double);
  CU(cudaFuncSetAttribute(variance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  variance_kernel<<<dim3(nslice, std::min(G, kGroupGrid), 6), kThreads, smem, st>>>(V); count_launch();
  variance_finish_kernel<<<(6 * F + 255) / 256, 256, 0, st>>>(n, F, nslice, d_m.p, d_div.p, d_partial.p, d_sigma2.p); count_launch();
  std::vector<double> sig(6 * (size_t)F), total(6);
  CU(cudaMemcpyAsync(sig.data(), d_sigma2.p, sig.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(total.data(), d_total.p, 6 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  // ---- fit points and initial values (host), the six fits (device) ------------------------------------------------------------
  FitArgs A; memset(&A, 0, sizeof A);
  std::vector<double> ptau, pl10;
  std::vector<std::vector<double>> fit_tau(6);
  for (int c = 0; c < 6; ++c) {
    curves.sigma2[c].assign(sig.begin() + (size_t)c * F, sig.begin() + (size_t)(c + 1) * F);
    std::vector<double> s2;
    if (c < 3) allan::accel_filter(curves.sigma2[c], curves.tau, s2, fit_tau[c]);   // FitAllanAcc::checkData
    else { s2 = curves.sigma2[c]; fit_tau[c] = curves.tau; }
    memset(&summary[c], 0, sizeof summary[c]);
    allan::init_value(s2, fit_tau[c], summary[c].init_coeffs, A.x0[c]);
    A.off[c] = (int)ptau.size();
    for (size_t i = 0; i < s2.size(); ++i) { ptau.push_back(fit_tau[c][i]); pl10.push_back(std::log(s2[i]) / std::log(10.0)); }
  }
  A.off[6] = (int)ptau.size();
  DevBuf<double> d_tau, d_l10, d_out;
  CU(d_tau.upload(ptau.data(), ptau.size(), st)); CU(d_l10.upload(pl10.data(), pl10.size(), st)); CU(d_out.alloc(6 * kFitOut));
  A.tau = d_tau.p; A.l10s = d_l10.p; A.out = d_out.p;
  fit_kernel<<<6, kThreads, 0, st>>>(A); count_launch();
  std::vector<double> out(6 * kFitOut);
  CU(cudaMemcpyAsync(out.data(), d_out.p, out.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  // ---- derived quantities (RunFit and the FitAllan* constructors' output) -------------------------------------------------------
  const int launches = kernel_launch_count() - launches0;
  const double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
  for (int c = 0; c < 6; ++c) {
    const double* f = &out[(size_t)c * kFitOut];
    const double* p = f;
    for (int q = 0; q < 5; ++q) params[5 * c + q] = p[q];
    curves.fit_deviation[c].resize(F);
    for (int i = 0; i < F; ++i) curves.fit_deviation[c][i] = std::sqrt(allan::model(p, curves.tau[i]));   // calcSimDeviation(taus)
    icc_allan_noise& z = noise[c]; memset(&z, 0, sizeof z);
    double dmin; int imin;
    min_deviation(p, fit_tau[c], dmin, imin);
    z.mean = total[c] / n;                                                       // getAvgValue (deg/h for the gyroscope), bit for bit
    z.bias_instability_tau = fit_tau[c].empty() ? 0.0 : fit_tau[c][imin];
    const double white = std::sqrt(freq) * std::sqrt(allan::model(p, 1));
    if (c < 3) { z.bias_instability = dmin; z.white_noise = white; }           // fitallan_acc.cc:111-117
    else {                                                                       // fitallan_gyr.cc:56-63, 115-121
      z.mean = z.mean / 3600;
      z.bias_b = std::sqrt(p[2] * p[2]) / 0.6642824703 / (57.3 * 3600);
      z.bias_instability = dmin / (57.3 * 3600);
      z.white_noise_n = std::sqrt(freq) * (std::sqrt(p[1] * p[1]) / 60.0) * 60 / 57.3;
      z.white_noise = white / (57.3 * 3600);
    }
    icc_allan_summary& S = summary[c];
    S.n_samples = n; S.n_factors = F; S.n_fit_points = A.off[c + 1] - A.off[c];
    S.iterations = (int)f[7]; S.termination = (int)f[8]; S.successful_steps = (int)f[9]; S.gpu_launches = launches;
    S.freq = freq; S.period = period; S.initial_cost = f[5]; S.final_cost = f[6]; S.seconds_total = seconds;
  }
  return ICC_OK;
}

}  // namespace icc
