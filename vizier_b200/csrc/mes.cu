// Max-value samples of MaxValueEntropySearch (acquisitions.py:293-365; Wang & Jegelka, ICML 2017, §3.1, and the
// authors' Gumbel-sampling code), drawn on the device once per fit (vzgp_mes_fit; DESIGN §6k):
//   1. mu_i, sd_i at the N valid trials through launch_score, the moments every scoring call computes;
//   2. k_mes_fit, one CTA: log P(y) = sum_i log Phi((y - mu_i) / sd_i) by a block reduction in a fixed order, the
//      degenerate test P(left) >= 0.25, the bracket, FIT_ITERS bisection steps for the three quartiles together, the
//      Gumbel fit, and the K samples written straight into the handle's fixed buffer.
// tests/mes_oracle.py::fit restates it.
#include "eagle_dev.cuh"

namespace vzgp {

namespace {

constexpr int kFitThreads = 256;
constexpr int kFitIters = 64;          // bisection halvings per quartile
constexpr int kBracketDoublings = 128;
__constant__ double kLogQ[3] = {-1.3862943611198906, -0.6931471805599453, -0.2876820724517809};   // log q
__constant__ double kLogLogQ[3] = {0.32663425997828094, -0.36651292058166435, -1.2458993237072382};   // log(-log q)

// log Phi(z) without log(normcdf(z)), which is -inf below z ~ -38.
__device__ __forceinline__ double log_ndtr(double z) {
  if (z < 0.0) return log(0.5 * erfcx(-z * 0.7071067811865476)) - 0.5 * z * z;
  return log1p(-0.5 * erfc(z * 0.7071067811865476));
}

// log P(y[j]) for j < CNT into out[j], the same value in every thread.  Thread t sums trials t, t + 256, ... in order,
// then a shared-memory tree adds the partial sums: the order is fixed, so the fit is deterministic.
template <int CNT>
__device__ __forceinline__ void block_log_p(const double* __restrict__ mu, const double* __restrict__ sd, int n,
                                            const double* y, double* out, double* red) {
  const int tid = threadIdx.x;
  double acc[CNT];
#pragma unroll
  for (int j = 0; j < CNT; ++j) acc[j] = 0.0;
  for (int i = tid; i < n; i += kFitThreads) {
    const double m = mu[i], s = sd[i];
#pragma unroll
    for (int j = 0; j < CNT; ++j) {
      const double z = s > 0.0 ? (y[j] - m) / s : (y[j] > m ? INFINITY : -INFINITY);   // sd = 0: the step y > mu
      acc[j] += log_ndtr(z);
    }
  }
#pragma unroll
  for (int j = 0; j < CNT; ++j) red[j * kFitThreads + tid] = acc[j];
  __syncthreads();
  for (int s = kFitThreads / 2; s > 0; s >>= 1) {
    if (tid < s)
#pragma unroll
      for (int j = 0; j < CNT; ++j) red[j * kFitThreads + tid] += red[j * kFitThreads + tid + s];
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < CNT; ++j) out[j] = red[j * kFitThreads];
  __syncthreads();
}

__global__ void __launch_bounds__(kFitThreads) k_mes_fit(const double* __restrict__ mu, const double* __restrict__ sd,
                                                         int n, double left, double floor_value, int K, uint64_t seed,
                                                         double* __restrict__ out) {
  __shared__ double red[3 * kFitThreads];
  const int tid = threadIdx.x;
  double y[3] = {left, left, left}, lp[3];
  block_log_p<1>(mu, sd, n, y, lp, red);
  if (lp[0] >= kLogQ[0]) {   // the authors' degenerate branch: P(left) >= 0.25
    for (int k = tid; k < K; k += kFitThreads) out[k] = floor_value;
    return;
  }
  double top = -INFINITY;
  for (int i = tid; i < n; i += kFitThreads) top = fmax(top, mu[i] + 5.0 * sd[i]);
  red[tid] = top;
  __syncthreads();
  for (int s = kFitThreads / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] = fmax(red[tid], red[tid + s]);
    __syncthreads();
  }
  double w = red[0] - left;
  __syncthreads();
  if (!(w > 0.0)) w = 1.0;
  for (int it = 0; it < kBracketDoublings; ++it) {
    y[0] = left + w;
    block_log_p<1>(mu, sd, n, y, lp, red);
    if (lp[0] >= kLogQ[2]) break;
    w *= 2.0;
  }
  double lo[3] = {left, left, left}, hi[3] = {left + w, left + w, left + w};
  for (int it = 0; it < kFitIters; ++it) {
#pragma unroll
    for (int j = 0; j < 3; ++j) y[j] = 0.5 * (lo[j] + hi[j]);
    block_log_p<3>(mu, sd, n, y, lp, red);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (lp[j] < kLogQ[j]) lo[j] = y[j];
      else hi[j] = y[j];
    }
  }
  double r[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) r[j] = 0.5 * (lo[j] + hi[j]);
  const double b = (r[2] - r[0]) / (kLogLogQ[0] - kLogLogQ[2]);
  const double a = r[1] - b * kLogLogQ[1];
  for (int k = tid; k < K; k += kFitThreads) {
    const double u = philox_uniform(seed, kStreamMes, 0, (uint64_t)k);
    out[k] = fmax(a - b * log(-log(u)), floor_value);
  }
}

}  // namespace

int launch_mes_fit(vzgp_handle* h, double best_label, int K, uint64_t seed) {
  const int n = h->n_valid;
  VZ_TRY(h->mes.reserve(sizeof(double) * kMaxMesSamples));
  VZ_TRY(h->mes_tmp.reserve(sizeof(double) * 3 * (size_t)n));
  double* score = h->mes_tmp.as<double>();
  double* mu = score + n;
  double* sd = mu + n;
  vzgp_acq acq = {};
  acq.use_trust_region = 0;
  acq.trust_radius = 1.0;
  // the trials are the first n_valid rows of the handle's padded copy
  VZ_TRY(launch_score(h, h->X.as<double>(), nullptr, n, &acq, score, mu, sd, nullptr, nullptr));
  k_mes_fit<<<1, kFitThreads, 0, h->stream>>>(mu, sd, n, best_label, best_label + 5.0 * sqrt(h->sn2), K, seed,
                                              h->mes.as<double>());
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
