// Parallel (q-) acquisitions: QEI, QPI and QUCB of sets of q points (acquisitions.py:495-568), estimated by Monte
// Carlo over each set's joint posterior predictive.
//
//   k_qset_moments  one CTA per set: mean mu = K* alpha + mean_const, the q x q block
//                   Sigma = k(x_i, x_j) + sn2 delta_ij - W_i . W_j from the chunk's explicit K* and W = K* L^-T
//                   (the general scoring route), and the L-inf distance of each point to the trusted trials.
//                   Only the block diagonal of the joint covariance is formed.
//   k_qacq_mc       one CTA per set: the Cholesky factor of every member's block with the jitter ladder of
//                   retrying_cholesky (tuned_gp_models.py:272-280), then S Philox draws f = mu + L z spread over the
//                   threads, each thread summing its draws in order and one fixed-shape block reduction, so a repeated
//                   call is bit-identical.  tests/qacq_oracle.py::qacq_score restates both kernels.
#include "eagle_dev.cuh"

namespace vzgp {

constexpr int kQMax = 16;              // points per set
constexpr int kQMaxSamples = 8192;
constexpr int kQMomThreads = 128;
constexpr int kQMcThreads = 256;
constexpr double kQeiExploration = 0.01;   // tfp_bo ParallelExpectedImprovement default exploration
constexpr double kQJitter = 1e-4;          // retrying_cholesky(jitter=1e-4, max_iters=5)
constexpr int kQMaxRetries = 5;

struct QMomArgs {
  const double* Ks;       // [mp x np] of this chunk
  const double* W;        // [mp x np]
  const double* Xs;       // [mp x dc] padded candidates of this chunk
  const int32_t* Zs;      // [mp x dk]
  const double* X;        // [np x dc] trials
  const double* alpha;
  int q, np, n_valid, dc, dk, want_linf;
  KernelParams kp;
  double sn2, mean_const;
  TrustRegion tr;
  double* mu;             // [sets * q] of this chunk
  double* cov;            // [sets][q][q]
  double* linf;           // [sets * q] or nullptr
};

// k(x_i, x_j) with the arithmetic of k_cross_kernel (tile_d2 / tile_lin): difference-first scaled distance, then the
// Hamming term, Matern-5/2, plus the linear term of the linear_coef model.
__device__ __forceinline__ double pair_kernel(const QMomArgs& a, int ri, int rj) {
  const double* xi = a.Xs + (size_t)ri * a.dc;
  const double* xj = a.Xs + (size_t)rj * a.dc;
  double d2 = 0.0, lin = 0.0;
  for (int d = 0; d < a.dc; ++d) {
    const double diff = xi[d] - xj[d];
    d2 = fma(diff * diff, a.kp.inv_ls2_c[d], d2);
  }
  for (int k = 0; k < a.dk; ++k)
    d2 += (a.Zs[(size_t)ri * a.dk + k] != a.Zs[(size_t)rj * a.dk + k]) ? a.kp.inv_ls2_k[k] : 0.0;
  double v = matern52(d2, a.kp.sf2);
  if (a.kp.use_linear) {
    for (int d = 0; d < a.dc; ++d) {
      const double w = a.kp.inv_ls_c[d];
      lin = fma(fma(xi[d], w, -a.kp.lin_b), fma(xj[d], w, -a.kp.lin_b), lin);
    }
    v = fma(a.kp.lin_a, lin, v);
  }
  return v;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Tasks of one set, one warp each: q means, q (q + 1) / 2 covariance entries (i >= j), q distances.
__global__ void __launch_bounds__(kQMomThreads) k_qset_moments(const QMomArgs a) {
  const int set = blockIdx.x, q = a.q, lane = threadIdx.x & 31;
  const int r0 = set * q, npairs = q * (q + 1) / 2;
  const int ntask = q + npairs + (a.want_linf ? q : 0);
  for (int t = threadIdx.x >> 5; t < ntask; t += kQMomThreads / 32) {
    if (t < q) {
      const double* ks = a.Ks + (size_t)(r0 + t) * a.np;
      double m = 0.0;
      for (int j = lane; j < a.n_valid; j += 32) m = fma(ks[j], a.alpha[j], m);
      m = warp_sum(m);
      if (lane == 0) a.mu[r0 + t] = m + a.mean_const;
    } else if (t < q + npairs) {
      int p = t - q, i = 0;
      while (p > i) { p -= i + 1; ++i; }
      const int j = p;
      const double* wi = a.W + (size_t)(r0 + i) * a.np;
      const double* wj = a.W + (size_t)(r0 + j) * a.np;
      double g = 0.0;
      for (int k = lane; k < a.np; k += 32) g = fma(wi[k], wj[k], g);
      g = warp_sum(g);
      if (lane == 0) {
        double c = pair_kernel(a, r0 + i, r0 + j) - g;
        if (i == j) c += a.sn2;
        a.cov[((size_t)set * q + i) * q + j] = c;
        a.cov[((size_t)set * q + j) * q + i] = c;
      }
    } else {
      const int row = r0 + (t - q - npairs);
      double dist = tr_lane_distance(a.tr, a.Xs + (size_t)row * a.dc, a.X, a.dc, lane);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dist = fmin(dist, __shfl_xor_sync(0xffffffffu, dist, o));
      if (lane == 0) a.linf[row] = dist;
    }
  }
}

struct QMcArgs {
  const double* mean;     // [E][n_sets * q]
  const double* cov;      // [E][n_sets][q][q]
  const double* linf;     // [n_sets * q] or nullptr (no trust region)
  int n_sets, q, E, S, period, kind;
  double best, coef;
  TrustRegion tr;
  uint64_t seed;
  double* score;
  double* mu;             // optional [n_sets * q]: mixture mean
  double* sigma;          // optional [n_sets * q]: mixture stddev
};

__device__ __forceinline__ double qacq_normal(uint64_t seed, uint64_t e) {
  const double u1 = philox_uniform(seed, kStreamQacqNormal, 0, 2 * e);
  const double u2 = philox_uniform(seed, kStreamQacqNormal, 0, 2 * e + 1);
  // cospi(2 u2) = cos(2 pi u2) without cos's large-argument reduction (and its stack frame)
  return sqrt(-2.0 * log(1.0 - u1)) * cospi(2.0 * u2);
}

// Dynamic shared memory: L [E][q][q] | member means [E][q] | mixture mean [q] | reduction [32].
__global__ void __launch_bounds__(kQMcThreads) k_qacq_mc(const QMcArgs a) {
  extern __shared__ double smem[];
  __shared__ int bad;
  const int set = blockIdx.x, q = a.q, E = a.E, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* L = smem;
  double* mus = L + (size_t)E * q * q;
  double* qmu = mus + E * q;
  double* red = qmu + q;
  if (threadIdx.x == 0) bad = 0;
  for (int i = threadIdx.x; i < E * q; i += blockDim.x) {
    const int e = i / q, j = i - e * q;
    mus[i] = a.mean[(size_t)e * a.n_sets * q + (size_t)set * q + j];
  }
  __syncthreads();
  // one warp per member: right-looking Cholesky of Sigma + shift I, lane = row, shifts 0, 1e-4, 1e-3, ...
  for (int e = warp; e < E; e += kQMcThreads / 32) {
    double* c = L + (size_t)e * q * q;
    const double* src = a.cov + ((size_t)e * a.n_sets + set) * q * q;
    bool ok = false;
    double shift = 0.0;
    for (int attempt = 0; attempt <= kQMaxRetries && !ok; ++attempt) {
      __syncwarp();
      for (int i = lane; i < q * q; i += 32) {
        const int r = i / q, col = i - r * q;
        c[i] = col <= r ? src[i] + (r == col ? shift : 0.0) : 0.0;
      }
      __syncwarp();
      ok = true;
      for (int k = 0; k < q; ++k) {
        const double d = c[k * q + k];
        if (!(d > 0.0) || !isfinite(d)) { ok = false; break; }
        const double l = sqrt(d);
        __syncwarp();
        if (lane == 0) c[k * q + k] = l;
        for (int i = k + 1 + lane; i < q; i += 32) c[i * q + k] /= l;
        __syncwarp();
        for (int i = k + 1 + lane; i < q; i += 32) {
          const double lik = c[i * q + k];
          for (int j = k + 1; j <= i; ++j) c[i * q + j] -= lik * c[j * q + k];
        }
        __syncwarp();
      }
      shift = shift == 0.0 ? kQJitter : shift * 10.0;
    }
    if (!ok && lane == 0) bad = 1;
  }
  if (threadIdx.x < q) {
    const int j = threadIdx.x;
    double s1 = 0.0, s2 = 0.0;
    for (int e = 0; e < E; ++e) {
      const double m = mus[e * q + j];
      s1 += m;
      s2 += a.cov[(((size_t)e * a.n_sets + set) * q + j) * q + j] + m * m;
    }
    // the mixture's mean and variance (stochastic_process_model.py:858-867); one member: its own diagonal
    const double mean = s1 / E;
    const double var = E == 1 ? a.cov[((size_t)set * q + j) * q + j] : s2 / E - mean * mean;
    qmu[j] = mean;
    if (a.mu) a.mu[(size_t)set * q + j] = mean;
    if (a.sigma) a.sigma[(size_t)set * q + j] = sqrt(fmax(var, 0.0));
  }
  __syncthreads();
  const uint64_t pos = (uint64_t)(set % a.period);
  const bool no_best = !isfinite(a.best);
  double acc = 0.0;
  for (int s = threadIdx.x; s < a.S; s += kQMcThreads) {
    const uint64_t ps = pos * (uint64_t)a.S + (uint64_t)s;
    int m = 0;
    if (E > 1) m = min((int)(philox_uniform(a.seed, kStreamQacqMember, 0, ps) * E), E - 1);
    const double* Lm = L + (size_t)m * q * q;
    double f[kQMax];
#pragma unroll
    for (int j = 0; j < kQMax; ++j) f[j] = j < q ? mus[m * q + j] : 0.0;
#pragma unroll
    for (int k = 0; k < kQMax; ++k) {
      if (k < q) {
        const double z = qacq_normal(a.seed, ps * (uint64_t)q + (uint64_t)k);
#pragma unroll
        for (int j = k; j < kQMax; ++j)
          if (j < q) f[j] = fma(Lm[j * q + k], z, f[j]);
      }
    }
    double v = -INFINITY;
    if (a.kind == VZGP_QACQ_QUCB) {
#pragma unroll
      for (int j = 0; j < kQMax; ++j)
        if (j < q) v = fmax(v, fma(a.coef, fabs(f[j] - qmu[j]), qmu[j]));
    } else {
#pragma unroll
      for (int j = 0; j < kQMax; ++j)
        if (j < q) v = fmax(v, f[j]);
      if (!no_best) v = a.kind == VZGP_QACQ_QEI ? fmax(v - a.best - kQeiExploration, 0.0) : (v - a.best > 0.0 ? 1.0 : 0.0);
    }
    acc += v;
  }
  const double total = block_sum(acc, red);
  if (threadIdx.x == 0) {
    double tr = 0.0;
    if (a.tr.apply)
      for (int j = 0; j < q; ++j) tr += tr_set_term(a.tr, a.linf[(size_t)set * q + j]);
    a.score[set] = bad ? NAN : total / a.S + tr;
  }
}

int launch_qacq_mc(vzgp_handle* h, int n_sets, int q, int E, const double* mean, const double* cov, const double* linf,
                   const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma) {
  if (n_sets <= 0) return 0;
  QMcArgs a;
  a.mean = mean; a.cov = cov; a.linf = linf;
  a.n_sets = n_sets; a.q = q; a.E = E; a.S = qa->num_samples;
  a.period = qa->period > 0 ? qa->period : n_sets;
  a.kind = qa->kind;
  a.tr = trust_region_of(h, *qa, false);
  a.tr.apply = linf != nullptr && tr_needs_distance(a.tr);
  a.best = qa->best_label; a.coef = qa->coefficient;
  a.seed = seed; a.score = score; a.mu = mu; a.sigma = sigma;
  const size_t sm = sizeof(double) * ((size_t)E * q * q + (size_t)E * q + q + 32);
  k_qacq_mc<<<n_sets, kQMcThreads, sm, h->stream>>>(a);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int launch_score_qsets(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int n_sets, int q,
                       const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma, double* linf) {
  if (n_sets <= 0) return 0;
  vzgp_handle* h0 = hs[0];
  const int M = n_sets * q, dc = h0->dc, dk = h0->dk;
  const TrustRegion tr = trust_region_of(h0, *qa, false);   // measured on member 0's trials
  const bool want_linf = linf != nullptr || tr_needs_distance(tr);
  const size_t nmean = (size_t)E * M, ncov = (size_t)E * M * q;
  // qmom: member means [E][M] | covariance blocks [E][n_sets][q][q] (unless the caller's cov_out) | distances [M]
  VZ_TRY(h0->qmom.reserve(sizeof(double) * (nmean + (qa->cov_out ? 0 : ncov) + M)));
  double* means = h0->qmom.as<double>();
  double* covs = qa->cov_out ? qa->cov_out : means + nmean;
  double* dist = linf ? linf : means + nmean + (qa->cov_out ? 0 : ncov);
  const int rows = (kGeneralChunk / q) * q;   // chunks of whole sets
  for (int e = 0; e < E; ++e) {
    vzgp_handle* h = hs[e];
    GeneralChunk c;
    VZ_TRY(general_chunk_buffers(h, &c));
    QMomArgs a;
    a.Ks = c.Ks; a.W = c.W; a.Xs = c.Xp; a.Zs = c.Zp; a.X = h->X.as<double>(); a.alpha = h->alpha.as<double>();
    a.q = q; a.np = h->np; a.n_valid = h->n_valid; a.dc = dc; a.dk = dk; a.kp = h->kp;
    a.sn2 = h->sn2; a.mean_const = h->mean_const;
    a.tr = tr;
    a.want_linf = (e == 0 && want_linf) ? 1 : 0;
    for (int m0 = 0; m0 < M; m0 += rows) {
      const int mc = M - m0 < rows ? M - m0 : rows;
      VZ_TRY(launch_general_chunk(h, dc > 0 ? Xs + (size_t)m0 * dc : Xs, dk > 0 ? Zs + (size_t)m0 * dk : Zs, mc, c));
      a.mu = means + (size_t)e * M + m0;
      a.cov = covs + ((size_t)e * M + m0) * q;
      a.linf = a.want_linf ? dist + m0 : nullptr;
      k_qset_moments<<<mc / q, kQMomThreads, 0, h->stream>>>(a);
      VZ_CHECK_LAUNCH();
      h->launches++;
    }
    h->score_route = VZGP_ROUTE_GENERAL;
  }
  return launch_qacq_mc(h0, n_sets, q, E, means, covs, want_linf ? dist : nullptr, qa, seed, score, mu, sigma);
}

}  // namespace vzgp
