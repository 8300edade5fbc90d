// Vectorised Eagle/Firefly acquisition optimiser: device-resident population state and the
// suggest / update / trim / top-k steps (continuous + categorical features, n_parallel == 1).
//
// Replaces (reference): VectorizedEagleStrategy.init_state/_populate_pool_with_prior_trials
// (vizier/_src/algorithms/optimizers/eagle_strategy.py:527-713), suggest/_create_features/
// _create_random_perturbations/_create_categorical_feature_logits (:720-1073),
// update/_update_pool_features_and_rewards/_trim_pool (:1075-1247), DefaultRandomSampler
// (:271-322) and VectorizedOptimizer._update_best_results
// (vizier/_src/algorithms/optimizers/vectorized_base.py:544-587).
// Randomness is Philox4x32-10 (see device.cuh); with n_parallel == 1 the reference's normalised
// Laplace perturbation of continuous features is exactly +-1 per coordinate
// (eagle_strategy.py:1033-1044); categorical logits get real Laplace noise and are sampled by
// Gumbel-max (= tfd.Categorical(logits).sample).  Element numbering of the draws is the contract
// shared with oracle/eagle_oracle.py.
#include <climits>

#include "device.cuh"
#include "eagle_dev.cuh"
#include "launchers.h"

namespace vzgp {

// ---------------------------------------------------------------------------
// init: pool <- Philox uniforms; rewards=-inf; perturbations=cfg.perturbation; best=-inf.
// ---------------------------------------------------------------------------
__global__ void k_eagle_init(EagleDev e) {
  const int64_t total = (int64_t)e.P * e.D;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < total; i += nth) e.pool[i] = philox_uniform(e.seed, kStreamInitPool, 0, (uint64_t)i);
  for (int64_t i = tid; i < (int64_t)e.P * e.Dk; i += nth)
    e.pool_z[i] = uniform_category(philox_uniform(e.seed, kStreamInitCat, 0, (uint64_t)i), e.sizes[i % e.Dk]);
  for (int64_t i = tid; i < e.P; i += nth) {
    e.rewards[i] = -INFINITY;
    e.pert[i] = e.cfg.perturbation;
  }
  if (blockIdx.x == 0) {
    for (int c = threadIdx.x; c < e.count; c += blockDim.x) {
      e.best_r[c] = -INFINITY;
      e.best_id[c] = LLONG_MAX;
    }
    for (int c = threadIdx.x; c < e.count * e.D; c += blockDim.x) e.best_x[c] = 0.0;
    for (int c = threadIdx.x; c < e.count * e.Dk; c += blockDim.x) e.best_z[c] = 0;
    if (threadIdx.x == 0) { *e.best_reward = -INFINITY; *e.iter = 0; }
  }
}


// ---------------------------------------------------------------------------
// Prior-trial seeding (single CTA; the reference loop is sequential too).
// prior [n x D] / prior_z [n x Dk] in creation order, prior_r [n] their acquisition values.
// ord [n] int workspace, chosen_r [left] workspace.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_eagle_seed_priors(EagleDev e, const double* __restrict__ prior,
                                                           const int32_t* __restrict__ prior_z,
                                                           const double* __restrict__ prior_r, int n,
                                                           int* __restrict__ ord,
                                                           double* __restrict__ chosen_r) {
  __shared__ double sv[256];
  __shared__ int si[256];
  const int tid = threadIdx.x, D = e.D, Dk = e.Dk;
  const int n_random = (int)(e.P * (1.0 - e.cfg.prior_trials_pool_pct));
  const int left = e.P - n_random;
  // _mask_flip: valid entries newest first, then the -inf ones (eagle_strategy.py:472-496).
  if (tid == 0) {
    int w = 0;
    for (int i = n - 1; i >= 0; --i)
      if (!(isinf(prior_r[i]) && prior_r[i] < 0)) ord[w++] = i;
    for (int i = n - 1; i >= 0; --i)
      if (isinf(prior_r[i]) && prior_r[i] < 0) ord[w++] = i;
  }
  __syncthreads();
  const int chosen = n < left ? n : left;
  double* feat = e.pool + (size_t)n_random * D;      // the chosen set lives directly in the pool
  int32_t* featz = e.pool_z + (size_t)n_random * Dk;
  for (int c = tid; c < chosen; c += 256) chosen_r[c] = prior_r[ord[c]];
  __syncthreads();
  // Entries whose reward is -inf (padded priors) keep the random row already in the pool
  // (eagle_strategy.py:693-702).
  for (int idx = tid; idx < chosen * D; idx += 256) {
    const int c = idx / D, d = idx % D;
    if (!(isinf(chosen_r[c]) && chosen_r[c] < 0)) feat[(size_t)c * D + d] = prior[(size_t)ord[c] * D + d];
  }
  for (int idx = tid; idx < chosen * Dk; idx += 256) {
    const int c = idx / Dk, d = idx % Dk;
    if (!(isinf(chosen_r[c]) && chosen_r[c] < 0)) featz[(size_t)c * Dk + d] = prior_z[(size_t)ord[c] * Dk + d];
  }
  __syncthreads();
  for (int i = left; i < n; ++i) {
    const double* x = prior + (size_t)ord[i] * D;
    const int32_t* z = prior_z + (size_t)ord[i] * Dk;
    double bv = INFINITY;
    int bi = INT_MAX;
    for (int c = tid; c < left; c += 256) {
      const double s = fly_distance(x, feat + (size_t)c * D, D, z, featz + (size_t)c * Dk, Dk);
      if (s < bv || (s == bv && c < bi)) { bv = s; bi = c; }
    }
    sv[tid] = bv; si[tid] = bi;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (tid < o) {
        if (sv[tid + o] < sv[tid] || (sv[tid + o] == sv[tid] && si[tid + o] < si[tid])) {
          sv[tid] = sv[tid + o]; si[tid] = si[tid + o];
        }
      }
      __syncthreads();
    }
    const int ind = si[0];
    const double ri = prior_r[ord[i]];
    const bool repl = chosen_r[ind] < ri;
    __syncthreads();
    if (repl) {
      for (int d = tid; d < D; d += 256) feat[(size_t)ind * D + d] = x[d];
      for (int d = tid; d < Dk; d += 256) featz[(size_t)ind * Dk + d] = z[d];
      if (tid == 0) chosen_r[ind] = ri;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) k_eagle_suggest(EagleDev e) {
  extern __shared__ double smem[];
  eagle_suggest_block<8>(e, blockIdx.x, smem);
}

__global__ void __launch_bounds__(256) k_eagle_update(EagleDev e) {
  extern __shared__ double smem[];
  eagle_update_block<false>(e, smem);
}

// ---------------------------------------------------------------------------
// Small studies (N <= 64 trials, batch <= 64): the WHOLE optimisation loop in one persistent CTA.
// The default designer runs 3000 sequential suggest -> score -> update iterations of 25 candidates
// (vectorized_base.py:431-495); as separate launches each iteration costs five kernels (~25 us even
// from a CUDA graph).  Here the model (L^-1, trial features, alpha) is staged in shared memory once,
// every iteration calls the same suggest/update code as the stand-alone kernels and scores the batch
// in place: K* tile -> W = K* L^-T on the DMMA pipe -> sigma^2, UCB, trust region.  Barriers are
// __syncthreads only; the population state stays in global memory (L1/L2 resident, written and read by
// this CTA alone).
// ---------------------------------------------------------------------------
constexpr int kPLD = 68;    // row stride of the two DMMA operands in smem (8-byte fragment loads conflict-free)
constexpr int kPXLD = 66;

constexpr int kPThreads = 1024;   // persistent kernel: 32 warps = one warp per batch fly (B <= 32) per pass

struct ModelSmem {   // one GP staged in shared memory (np == 64)
  double* linv;    // [64][kPLD]
  double* xt;      // [dc][kPXLD] trial features (unscaled), transposed
  double* alpha;   // [64]
  int32_t* z;      // [dk][kPXLD]
};
struct PersistSmem {
  double* eagle;   // suggest / update scratch
  ModelSmem a, b;  // b only with the GP-UCB-PE acquisition
  double* ks;      // [64][kPLD] K* tile of the model being evaluated
  double* cand;    // [dc][kPXLD] candidates, transposed
  double* mu;      // [2][64] posterior mean of model a / b
  double* sd;      // [2][64] posterior stddev
  double* linf;    // [64] trust-region distance (model a for UCB, model b for UCB-PE)
  double* rs4;     // [4][64] partial row sums of W^2
  int32_t* cz;     // [dk][kPXLD]
};

__device__ __forceinline__ void stage_model64(const SmallModel& m, const ModelSmem& ms) {
  const int tid = threadIdx.x, dc = m.kp.dc, dk = m.kp.dk;
  for (int i = tid; i < 64 * 64; i += kPThreads) ms.linv[(i >> 6) * kPLD + (i & 63)] = m.Linv[i];
  for (int i = tid; i < dc * 64; i += kPThreads) ms.xt[(i >> 6) * kPXLD + (i & 63)] = m.XTu[i];
  for (int i = tid; i < 64 * dk; i += kPThreads) {
    const int r = i / dk, k = i - r * dk;
    ms.z[k * kPXLD + r] = m.Z[i];
  }
  if (tid < 64) ms.alpha[tid] = m.alpha[tid];
}

// Candidates of the current batch, transposed into shared memory (ends with a barrier).
__device__ __forceinline__ void stage_candidates64(const PersistSmem& sm, int dc, int dk, const double* cand,
                                                   const int32_t* candz, int B) {
  const int tid = threadIdx.x;
  for (int e = tid; e < 64 * dc; e += kPThreads) {
    const int r = e / dc, d = e - r * dc;
    sm.cand[d * kPXLD + r] = r < B ? cand[(size_t)r * dc + d] : 0.0;
  }
  for (int e = tid; e < 64 * dk; e += kPThreads) {
    const int r = e / dk, k = e - r * dk;
    sm.cz[k * kPXLD + r] = r < B ? candz[(size_t)r * dk + k] : -1;
  }
  __syncthreads();
}

// Posterior of one staged model at the staged candidates: mu_out[i], sd_out[i] and (if linf_out) the
// trust-region distance to the first tr_rows trials.  Ends with a barrier.
__device__ __forceinline__ void posterior_tile64(const SmallModel& m, const ModelSmem& ms, const PersistSmem& sm,
                                                 int B, const SmallAcq& q, double* mu_out, double* sd_out,
                                                 double* linf_out, int* clamp_count) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int dc = m.kp.dc, dk = m.kp.dk;
  const bool want_linf = linf_out != nullptr;
  // ---- K* tile, mean, trust-region distance: thread = (candidate i, 4 trials) ----
  {
    const int i = tid >> 4, j0 = (tid & 15) * 4;
    double d2[4], lf[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) { d2[c] = 0.0; lf[c] = 0.0; }
    if ((i & ~1) >= B) {              // both candidate rows of this warp are padding
#pragma unroll
      for (int c = 0; c < 4; ++c) sm.ks[i * kPLD + j0 + c] = 0.0;
    } else {
      if (i < B) {
        for (int d = 0; d < dc; ++d) {
          const double av = sm.cand[d * kPXLD + i], w = m.kp.inv_ls2_c[d];
          const bool in_tr = want_linf && q.tr.mask[d];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const double df = av - ms.xt[d * kPXLD + j0 + c];
            d2[c] = fma(df * df, w, d2[c]);
            if (in_tr) lf[c] = fmax(lf[c], fabs(df));
          }
        }
        for (int k = 0; k < dk; ++k) {
          const int av = sm.cz[k * kPXLD + i];
          const double w = m.kp.inv_ls2_k[k];
#pragma unroll
          for (int c = 0; c < 4; ++c) d2[c] += (av != ms.z[k * kPXLD + j0 + c]) ? w : 0.0;
        }
      }
      double mu = 0.0, lmin = INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = j0 + c;
        const double kv = (i < B && j < m.n_valid) ? matern52(d2[c], m.kp.sf2) : 0.0;
        sm.ks[i * kPLD + j] = kv;
        mu = fma(kv, ms.alpha[j], mu);
        if (j < q.tr.rows) lmin = fmin(lmin, lf[c]);
      }
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        mu += __shfl_xor_sync(0xffffffffu, mu, o);
        lmin = fmin(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
      }
      if ((tid & 15) == 0) {
        mu_out[i] = mu;
        if (want_linf) linf_out[i] = lmin;
      }
    }
  }
  __syncthreads();
  // ---- W = K* Linv^T (lower triangular: k <= j), row sums of W^2.  Warp = (8 candidates, 2 column
  // tiles nt and 7 - nt: balanced triangular work); partial row sums combined through smem ----
  {
    const int mt = warp >> 2, pr = warp & 3;          // 8 m-tiles x 4 column-tile pairs
    if (mt * 8 < B) {
      const int fr = lane >> 2, fk = lane & 3;
      const double* Ar = sm.ks + (mt * 8 + fr) * kPLD + fk;
      double rsum = 0.0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int nt = h == 0 ? pr : 7 - pr;
        const double* Br = ms.linv + (nt * 8 + fr) * kPLD + fk;
        double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
        for (int ks = 0; ks < 2 * nt + 2; ks += 2) {
          dmma_8x8x4(a0, a1, Ar[4 * ks], Br[4 * ks]);
          dmma_8x8x4(b0, b1, Ar[4 * ks + 4], Br[4 * ks + 4]);
        }
        const double w0 = a0 + b0, w1 = a1 + b1;
        rsum = fma(w0, w0, rsum);
        rsum = fma(w1, w1, rsum);
      }
      rsum += __shfl_xor_sync(0xffffffffu, rsum, 1);
      rsum += __shfl_xor_sync(0xffffffffu, rsum, 2);
      if (fk == 0) sm.rs4[pr * 64 + mt * 8 + fr] = rsum;
    }
  }
  __syncthreads();
  if (tid < B) {
    const double rs = (sm.rs4[tid] + sm.rs4[64 + tid]) + (sm.rs4[128 + tid] + sm.rs4[192 + tid]);
    double var = m.kp.sf2 - rs + m.sn2;
    if (var < 0.0) { var = 0.0; atomicAdd(clamp_count, 1); }
    sd_out[tid] = sqrt(var);
  }
  __syncthreads();
}

// Acquisition of the batch from the staged model(s): acquisition function (acq_fn.cuh) + trust region (acquisitions.py:152-225) or the
// GP-UCB-PE combination of models a (completed trials) and b (completed + pending), gp_ucb_pe.py:344-492.
template <bool GENERIC>
__device__ __forceinline__ void score_batch64(const SmallModel& ma, const SmallModel& mb, const SmallAcq& q,
                                              const PersistSmem& sm, const double* cand, const int32_t* candz, int B,
                                              double* out_score, int* clamp_count) {
  const int tid = threadIdx.x;
  stage_candidates64(sm, ma.kp.dc, ma.kp.dk, cand, candz, B);
  if (q.pe_mode < 0) {
    posterior_tile64(ma, sm.a, sm, B, q, sm.mu, sm.sd, q.want_linf ? sm.linf : nullptr, clamp_count);
    if (tid < B) out_score[tid] = tr_apply(q.tr, acq_eval<GENERIC>(q.fn, sm.mu[tid], sm.sd[tid]), sm.linf[tid]);
  } else {
    posterior_tile64(ma, sm.a, sm, B, q, sm.mu, sm.sd, nullptr, clamp_count);
    posterior_tile64(mb, sm.b, sm, B, q, sm.mu + 64, sm.sd + 64, q.want_linf ? sm.linf : nullptr, clamp_count);
    if (tid < B) {
      double acq;
      if (q.pe_mode == 0) {
        acq = fma(q.coef, sm.sd[64 + tid], sm.mu[tid]);
      } else {
        const double explore_ucb = fma(sm.sd[tid], q.explore, sm.mu[tid]);
        acq = sm.sd[64 + tid] + q.penalty * fmin(explore_ucb - q.threshold, 0.0);
      }
      out_score[tid] = tr_apply(q.tr, acq, sm.linf[tid]);
    }
  }
  __syncthreads();
}

template <bool GENERIC>
__global__ void __launch_bounds__(kPThreads) k_eagle_persistent64(const EagleDev eg, SmallModel m, SmallModel mb,
                                                                  SmallAcq q, int steps, size_t eagle_scratch_doubles,
                                                                  int* clamp_count) {
  extern __shared__ double smem[];
  const int tid = threadIdx.x;
  const int dc = m.kp.dc, dk = m.kp.dk;
  const bool two = q.pe_mode >= 0;
  PersistSmem sm;
  double* p = smem;
  sm.eagle = p; p += eagle_scratch_doubles;
  sm.a.linv = p; p += 64 * kPLD;
  sm.a.xt = p; p += dc * kPXLD;
  sm.a.alpha = p; p += 64;
  sm.b.linv = p; p += two ? 64 * kPLD : 0;
  sm.b.xt = p; p += two ? dc * kPXLD : 0;
  sm.b.alpha = p; p += two ? 64 : 0;
  sm.ks = p; p += 64 * kPLD;
  sm.cand = p; p += dc * kPXLD;
  sm.mu = p; p += 128;
  sm.sd = p; p += 128;
  sm.linf = p; p += 64;
  sm.rs4 = p; p += 256;
  int32_t* ip0 = reinterpret_cast<int32_t*>(p);
  sm.a.z = ip0; ip0 += dk * kPXLD;
  sm.b.z = ip0; ip0 += two ? dk * kPXLD : 0;
  sm.cz = ip0; ip0 += dk * kPXLD;
  ip0 += (reinterpret_cast<uintptr_t>(ip0) & 7) ? 1 : 0;
  stage_model64(m, sm.a);
  if (two) stage_model64(mb, sm.b);
  // The population state moves into shared memory for the duration of the loop (generic pointers:
  // suggest / update run unchanged); every iteration would otherwise pay several dependent L2 round
  // trips for data this CTA wrote a moment ago.  best_* / tmp_* (touched once per step) stay global.
  __shared__ EagleDev es;      // the same descriptor with the state pointers redirected to shared memory
  if (tid == 0) {
    es = eg;
    double* p = reinterpret_cast<double*>(ip0);
    es.pool = p; p += (size_t)eg.P * eg.D;
    es.rewards = p; p += eg.P;
    es.pert = p; p += eg.P;
    es.best_reward = p; p += 2;
    es.batch = p; p += (size_t)eg.B * eg.D;
    es.batch_r = p; p += eg.B;
    int32_t* ip = reinterpret_cast<int32_t*>(p);
    es.iter = ip; ip += 4;
    es.pool_z = ip; ip += (size_t)eg.P * eg.Dk;
    es.batch_z = ip;
  }
  __syncthreads();
  const EagleDev& e = es;
  for (int i = tid; i < e.P * e.D; i += kPThreads) e.pool[i] = eg.pool[i];
  for (int i = tid; i < e.P; i += kPThreads) { e.rewards[i] = eg.rewards[i]; e.pert[i] = eg.pert[i]; }
  for (int i = tid; i < e.P * e.Dk; i += kPThreads) e.pool_z[i] = eg.pool_z[i];
  if (tid == 0) { *e.best_reward = *eg.best_reward; *e.iter = *eg.iter; }
  __syncthreads();
  constexpr int kW = kPThreads / 32;
  const int nvb = (e.B + kW - 1) / kW;
#ifdef VZ_EAGLE_TIMING
  long long c_s = 0, c_c = 0, c_u = 0, t0, t1;
#define VZ_ET(acc) do { t1 = clock64(); acc += t1 - t0; t0 = t1; } while (0)
  t0 = clock64();
#else
#define VZ_ET(acc) do {} while (0)
#endif
  for (int it = 0; it < steps; ++it) {
    for (int vb = 0; vb < nvb; ++vb) eagle_suggest_block<kW>(e, vb, sm.eagle);
    __syncthreads();
    VZ_ET(c_s);
    score_batch64<GENERIC>(m, mb, q, sm, e.batch, e.batch_z, e.B, e.batch_r, clamp_count);
    VZ_ET(c_c);
    if (tid < 256) eagle_update_block<true>(e, sm.eagle);
    __syncthreads();
    VZ_ET(c_u);
  }
  for (int i = tid; i < e.P * e.D; i += kPThreads) eg.pool[i] = e.pool[i];
  for (int i = tid; i < e.P; i += kPThreads) { eg.rewards[i] = e.rewards[i]; eg.pert[i] = e.pert[i]; }
  for (int i = tid; i < e.P * e.Dk; i += kPThreads) eg.pool_z[i] = e.pool_z[i];
  if (tid == 0) { *eg.best_reward = *e.best_reward; *eg.iter = *e.iter; }
#ifdef VZ_EAGLE_TIMING
  if (tid == 0) printf("eagle persistent: steps %d, cycles/step suggest %lld score %lld update %lld\n", steps,
                       c_s / steps, c_c / steps, c_u / steps);
#endif
}

// Z[m, k] = uniform category of feature k for candidate index_base+m (RandomVectorizedStrategy).
struct CatSizes { int v[kMaxDk]; };
__global__ void k_random_pool_cat(int32_t* __restrict__ Z, int64_t total, int dk, CatSizes sizes,
                                  int64_t elem_base, uint64_t seed, uint32_t stream) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; e < total; e += stride)
    Z[e] = uniform_category(philox_uniform(seed, stream, 0, (uint64_t)(elem_base + e)), sizes.v[(elem_base + e) % dk]);
}

__global__ void k_gather_rows_i32(const int32_t* __restrict__ Z, int dk, const long long* __restrict__ idx,
                                  int count, int64_t M, int32_t* __restrict__ out) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count * dk) return;
  int c = e / dk, d = e % dk;
  long long i = idx[c];
  out[e] = (i >= 0 && i < M) ? Z[(size_t)i * dk + d] : 0;
}

// ---------------------------------------------------------------------------
int launch_eagle_init(vzgp_handle* h, const EagleDev& e) {
  k_eagle_init<<<64, 256, 0, h->stream>>>(e);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_eagle_seed_priors(vzgp_handle* h, const EagleDev& e, const double* prior, const int32_t* prior_z,
                             const double* prior_r, int n, int* ord, double* chosen_r) {
  k_eagle_seed_priors<<<1, 256, 0, h->stream>>>(e, prior, prior_z, prior_r, n, ord, chosen_r);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
size_t eagle_suggest_smem(const EagleDev& e) {
  return sizeof(double) * (size_t)8 * (e.P + e.D) + sizeof(int32_t) * 8 * (size_t)(e.Dk + 2);
}
size_t eagle_suggest_cta_smem(const EagleDev& e) {
  return sizeof(double) * ((size_t)e.P + e.D + 8 * (size_t)(e.D + 2) + 4 + 64) + sizeof(int32_t) * (size_t)(e.Dk + 2 + 16) + 16;
}
size_t eagle_update_smem(const EagleDev& e) {
  return sizeof(double) * (size_t)(e.B + e.count) + (size_t)(e.B + e.count) + 16;
}
int eagle_prepare(const EagleDev& e) {
  VZ_TRY(raise_dyn_smem((const void*)k_eagle_suggest, eagle_suggest_smem(e)));
  VZ_TRY(raise_dyn_smem((const void*)k_eagle_update, eagle_update_smem(e)));
  return 0;
}
int launch_eagle_suggest(vzgp_handle* h, const EagleDev& e) {
  k_eagle_suggest<<<(e.B + 7) / 8, 256, eagle_suggest_smem(e), h->stream>>>(e);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_eagle_update(vzgp_handle* h, const EagleDev& e) {
  k_eagle_update<<<1, 256, eagle_update_smem(e), h->stream>>>(e);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
static size_t eagle_persistent_state_bytes(const EagleDev& e) {
  return sizeof(double) * ((size_t)e.P * e.D + 2 * (size_t)e.P + 2 + (size_t)e.B * e.D + e.B) +
         sizeof(int32_t) * (4 + (size_t)e.P * e.Dk + (size_t)e.B * e.Dk) + 16;
}

bool eagle_persistent_eligible(const vzgp_handle* h, const vzgp_handle* hB, const EagleDev& e) {
  static const bool enabled = [] { const char* v = getenv("VZGP_EAGLE_PERSISTENT"); return !(v && v[0] == '0'); }();
  const bool linear = h->kp.use_linear || (hB != nullptr && hB->kp.use_linear);   // in-kernel scoring knows Matern only
  return enabled && !linear && h->np == 64 && (hB == nullptr || hB->np == 64) && e.B <= 64 &&
         eagle_persistent_state_bytes(e) <= 64 * 1024;
}

static SmallModel small_model_of(const vzgp_handle* h) {
  SmallModel m;
  m.XTu = h->XT.as<double>() + (size_t)h->dc * h->np;
  m.Z = h->Z.as<int32_t>();
  m.Linv = h->Linv.as<double>();
  m.alpha = h->alpha.as<double>();
  m.kp = h->kp; m.sn2 = h->sn2; m.n_valid = h->n_valid;
  return m;
}

// acq (UCB on h) or pe (GP-UCB-PE on h = model A and hB = model B): exactly one is non-null.
int launch_eagle_persistent64(vzgp_handle* h, vzgp_handle* hB, const EagleDev& e, const vzgp_acq* acq,
                              const vzgp_pe_params* pe, int steps, const AcqFn* fn) {
  const SmallModel m = small_model_of(h);
  const SmallModel mb = hB ? small_model_of(hB) : m;
  SmallAcq q;
  memset(&q, 0, sizeof(q));
  if (pe) {   // GP-UCB-PE: the trust region is measured on model B's trials
    q.pe_mode = pe->mode; q.coef = pe->ucb_coefficient; q.explore = pe->explore_coefficient;
    q.penalty = pe->penalty_coefficient; q.threshold = pe->threshold;
    q.tr = trust_region_of(hB, *pe, true);
  } else {
    q.pe_mode = -1; q.fn = acq_fn_of(acq, fn);
    q.tr = trust_region_of(h, *acq, acq->tr_strict);
  }
  q.want_linf = tr_needs_distance(q.tr) ? 1 : 0;
  const size_t es = sizeof(double) * (size_t)(kPThreads / 32) * (e.P + e.D) + sizeof(int32_t) * (kPThreads / 32) * (size_t)(e.Dk + 2);
  const size_t eu = eagle_update_smem(e);
  const size_t scratch = ((es > eu ? es : eu) + 15) / 16 * 2;   // doubles, 16-byte multiple
  const int nm = pe ? 2 : 1;
  const size_t sm = sizeof(double) * (scratch + (size_t)(nm + 1) * 64 * kPLD + (size_t)(nm + 1) * h->dc * kPXLD +
                                      (size_t)nm * 64 + 128 + 128 + 64 + 256) +
                    sizeof(int32_t) * ((size_t)(nm + 1) * h->dk * kPXLD + 2) + eagle_persistent_state_bytes(e);
  if (sm > 227 * 1024) { set_error("persistent eagle kernel needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
  if (q.pe_mode < 0 && !acq_fn_is_ucb(q.fn)) {
    VZ_TRY(raise_dyn_smem((const void*)k_eagle_persistent64<true>, sm));
    k_eagle_persistent64<true><<<1, kPThreads, sm, h->stream>>>(e, m, mb, q, steps, scratch, h->small.as<int>());
  } else {
    VZ_TRY(raise_dyn_smem((const void*)k_eagle_persistent64<false>, sm));
    k_eagle_persistent64<false><<<1, kPThreads, sm, h->stream>>>(e, m, mb, q, steps, scratch, h->small.as<int>());
  }
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int launch_random_fill_cat(vzgp_handle* h, int32_t* Z, int64_t M, int dk, const int* sizes, int64_t index_base,
                           uint64_t seed, uint32_t stream) {
  const int64_t total = M * dk;
  if (total <= 0) return 0;
  CatSizes cs;
  for (int k = 0; k < kMaxDk; ++k) cs.v[k] = k < dk ? sizes[k] : 1;
  int64_t blocks = (total + 255) / 256;
  if (blocks > (int64_t)h->sm_count * 16) blocks = (int64_t)h->sm_count * 16;
  k_random_pool_cat<<<(unsigned)blocks, 256, 0, h->stream>>>(Z, total, dk, cs, index_base * dk, seed, stream);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_gather_rows_i32(vzgp_handle* h, const int32_t* Z, int dk, const long long* idx, int count, int64_t M,
                           int32_t* out) {
  if (count * dk == 0) return 0;
  k_gather_rows_i32<<<(count * dk + 255) / 256, 256, 0, h->stream>>>(Z, dk, idx, count, M, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
