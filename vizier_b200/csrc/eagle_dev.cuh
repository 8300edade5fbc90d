// Device-side pieces of the Eagle/Firefly optimiser shared by eagle.cu (stand-alone kernels and the
// single-CTA persistent loop) and eagle_grid.cu (the multi-CTA persistent loop).  See eagle.cu for the
// reference citations.
#pragma once
#include <climits>

#include "device.cuh"
#include "launchers.h"

namespace vzgp {

constexpr uint32_t kStreamInitCat = 4, kStreamCatLaplace = 5, kStreamCatGumbel = 6, kStreamTrimCat = 7,
                   kStreamPullRand = 9, kStreamPushRand = 10, kStreamSetLaplace = 11;
// Monte Carlo draws of the q-acquisitions (score_q.cu): Box-Muller normals and mixture members.
constexpr uint32_t kStreamQacqNormal = 12, kStreamQacqMember = 13;

__device__ __forceinline__ double laplace_from_uniform(double u) {
  const double v = u - 0.5;
  const double l = -log(fmax(1.0 - 2.0 * fabs(v), 1.1102230246251565e-16));
  return v > 0.0 ? l : (v < 0.0 ? -l : 0.0);
}
__device__ __forceinline__ double gumbel_from_uniform(double u) { return -log(-log(fmax(u, 1e-300))); }
// Continuous perturbation of coordinate d of batch fly b (eagle_strategy.py:1013-1046): Laplace noise divided by its
// largest magnitude over the q members of the same feature.  q = 1: the quotient is +-1 and one sign bit is drawn
// (stream kStreamPerturbSign); q > 1: coordinate d = m * Dm + f, uniforms of stream kStreamSetLaplace.
__device__ __forceinline__ double eagle_perturbation(const EagleDev& e, int t, int b, int d, double pert) {
  if (e.q <= 1) {
    const double u = philox_uniform(e.seed, kStreamPerturbSign, (uint32_t)t, (uint64_t)b * e.D + d);
    return u >= 0.5 ? pert : -pert;
  }
  const int dm = e.D / e.q, f = d % dm;
  double mine = 0.0, big = 0.0;
  for (int m = 0; m < e.q; ++m) {
    const int dd = m * dm + f;
    const double l = laplace_from_uniform(philox_uniform(e.seed, kStreamSetLaplace, (uint32_t)t, (uint64_t)b * e.D + dd));
    big = fmax(big, fabs(l));
    if (dd == d) mine = l;
  }
  return big > 0.0 ? mine / big * pert : 0.0;
}
__device__ __forceinline__ int uniform_category(double u, int size) {
  const int c = (int)(u * (double)size);
  return c < size - 1 ? c : size - 1;
}

// squared distance + Hamming distance (eagle_strategy.py:421-469)
__device__ __forceinline__ double fly_distance(const double* a, const double* b, int D, const int32_t* za,
                                               const int32_t* zb, int Dk) {
  double s = 0.0;
  for (int d = 0; d < D; ++d) {
    const double df = a[d] - b[d];
    s = fma(df, df, s);
  }
  for (int k = 0; k < Dk; ++k) s += (za[k] != zb[k]) ? 1.0 : 0.0;
  return s;
}

// ---------------------------------------------------------------------------
// suggest: one warp per batch fly, 8 flies per CTA.  Dynamic smem: 8*P doubles (forces) +
// 8*D doubles (the flies' own continuous features) + 8*Dk ints.
// ---------------------------------------------------------------------------
template <int NWARPS>
__device__ __forceinline__ void eagle_suggest_block(const EagleDev& e, int vblock, double* smem) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int P = e.P, B = e.B, D = e.D, Dk = e.Dk;
  const int t = *e.iter;
  const int nb = P / B;
  const int start = (t % nb) * B;
  const int b = vblock * NWARPS + warp;
  if (b >= B) return;
  const int i = start + b;
  double* s_f = smem + (size_t)warp * P;
  double* s_x = smem + (size_t)NWARPS * P + warp * D;
  int32_t* s_z = reinterpret_cast<int32_t*>(smem + (size_t)NWARPS * P + NWARPS * D) + warp * Dk;
  for (int d = lane; d < D; d += 32) s_x[d] = e.pool[(size_t)i * D + d];
  for (int d = lane; d < Dk; d += 32) s_z[d] = e.pool_z[(size_t)i * Dk + d];
  __syncwarp();
  double* out = e.batch + (size_t)b * D;
  int32_t* outz = e.batch_z + (size_t)b * Dk;
  if (t < nb) {  // still initialising: return the pool features (projected)
    for (int d = lane; d < D; d += 32) out[d] = fmin(fmax(s_x[d], 0.0), 1.0);
    for (int d = lane; d < Dk; d += 32) outz[d] = s_z[d];
    return;
  }
  const double ri = e.rewards[i];
  const double cexp = -e.cfg.visibility / (double)e.norm_dim * 10.0;
  int npull = 0, npush = 0;
  for (int j = lane; j < P; j += 32) {
    const double d2 = fly_distance(s_x, e.pool + (size_t)j * D, D, s_z, e.pool_z + (size_t)j * Dk, Dk);
    const double rj = e.rewards[j];
    const double dir = rj - ri;
    const double sd = (dir >= 0.0) ? e.cfg.gravity : -e.cfg.negative_gravity;
    const double f = sd * exp(cexp * d2) * (isfinite(rj) ? 1.0 : 0.0);
    s_f[j] = f;
    npull += (f > 0.0);
    npush += (f < 0.0);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    npull += __shfl_xor_sync(0xffffffffu, npull, o);
    npush += __shfl_xor_sync(0xffffffffu, npush, o);
  }
  __syncwarp();
  if (e.cfg.mutate_normalization_type == 1) {
    // RANDOM normalisation (eagle_strategy.py:858-885): random convex weights over the pulling
    // flies.  The reference masks BOTH weight matrices with (pull > 0), so pushes end up with zero
    // weight (reproduced).  Deliberate deviation: a fly that nobody pulls gets 0/0 = NaN weights
    // in the reference (NaN candidate, NaN best_reward from then on); here its weights are 0.
    double s1 = 0.0, s2 = 0.0;
    for (int j = lane; j < P; j += 32) {
      const double pos = s_f[j] > 0.0 ? 1.0 : 0.0;
      s1 += philox_uniform(e.seed, kStreamPullRand, (uint32_t)t, (uint64_t)b * P + j) * pos;
      s2 += philox_uniform(e.seed, kStreamPushRand, (uint32_t)t, (uint64_t)b * P + j) * pos;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    for (int j = lane; j < P; j += 32) {
      const double f = s_f[j];
      const double pos = f > 0.0 ? 1.0 : 0.0;
      const double w1 = s1 > 0.0 ? philox_uniform(e.seed, kStreamPullRand, (uint32_t)t, (uint64_t)b * P + j) * pos / s1 : 0.0;
      const double w2 = s2 > 0.0 ? philox_uniform(e.seed, kStreamPushRand, (uint32_t)t, (uint64_t)b * P + j) * pos / s2 : 0.0;
      s_f[j] = e.cfg.normalization_scale * fmax(f, 0.0) * w1 + e.cfg.normalization_scale * fmin(f, 0.0) * w2;
    }
  } else {
    const double wpull = npull > 0 ? e.cfg.normalization_scale / (double)npull : 0.0;
    const double wpush = npush > 0 ? e.cfg.normalization_scale / (double)npush : 0.0;
    // convert the forces to the normalised scale in place
    for (int j = lane; j < P; j += 32) {
      const double f = s_f[j];
      s_f[j] = f > 0.0 ? f * wpull : (f < 0.0 ? f * wpush : 0.0);
    }
  }
  __syncwarp();
  // ---- continuous features: lane handles dims lane and lane+32 ----
  // Four independent partial sums (j = 4q + r): the loop is a latency chain of loads and FMAs otherwise.
  double acc0 = 0.0, acc1 = 0.0, ssum = 0.0;
  const int d0 = lane, d1 = lane + 32;
  {
    double a0[4] = {0.0, 0.0, 0.0, 0.0}, a1[4] = {0.0, 0.0, 0.0, 0.0}, ss[4] = {0.0, 0.0, 0.0, 0.0};
    const bool wide = D > 32;
    int j = 0;
    for (; j + 4 <= P; j += 4) {
      double sc[4], p0[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        sc[r] = s_f[j + r];
        p0[r] = d0 < D ? e.pool[(size_t)(j + r) * D + d0] : 0.0;
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        ss[r] += sc[r];
        a0[r] = fma(sc[r], p0[r], a0[r]);
      }
      if (wide) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (d1 < D) a1[r] = fma(sc[r], e.pool[(size_t)(j + r) * D + d1], a1[r]);
      }
    }
    for (; j < P; ++j) {
      const double sc = s_f[j];
      ss[0] += sc;
      if (d0 < D) a0[0] = fma(sc, e.pool[(size_t)j * D + d0], a0[0]);
      if (d1 < D) a1[0] = fma(sc, e.pool[(size_t)j * D + d1], a1[0]);
    }
    acc0 = (a0[0] + a0[1]) + (a0[2] + a0[3]);
    acc1 = (a1[0] + a1[1]) + (a1[2] + a1[3]);
    ssum = (ss[0] + ss[1]) + (ss[2] + ss[3]);
  }
  const double pert = e.pert[i];
  if (d0 < D) {
    const double v = s_x[d0] + (acc0 - s_x[d0] * ssum) + eagle_perturbation(e, t, b, d0, pert);
    out[d0] = fmin(fmax(v, 0.0), 1.0);
  }
  if (d1 < D) {
    const double v = s_x[d1] + (acc1 - s_x[d1] * ssum) + eagle_perturbation(e, t, b, d1, pert);
    out[d1] = fmin(fmax(v, 0.0), 1.0);
  }
  // ---- categorical features (eagle_strategy.py:936-1011): lane = category (and lane+32) ----
  const double factor = D > 0 ? e.cfg.categorical_perturbation_factor : e.cfg.pure_categorical_perturbation_factor;
  const double log_same = Dk > 0 ? log(e.cfg.prob_same_category_without_perturbation) : 0.0;
  for (int k = 0; k < Dk; ++k) {
    const int size = e.sizes[k];
    if (size <= 1) {
      if (lane == 0) outz[k] = 0;
      continue;
    }
    const double log_diff = log((1.0 - e.cfg.prob_same_category_without_perturbation) / ((double)size - 1.0));
    double best_v = -INFINITY;
    int best_c = INT_MAX;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int c = lane + 32 * half;
      if (c < size) {
        double lg = 0.0;
        for (int j = 0; j < P; ++j) lg += (e.pool_z[(size_t)j * Dk + k] == c) ? s_f[j] : 0.0;
        lg += log_diff;
        if (c == s_z[k]) lg += -ssum + log_same - log_diff;
        const uint64_t el = ((uint64_t)b * Dk + k) * e.smax + c;
        lg += laplace_from_uniform(philox_uniform(e.seed, kStreamCatLaplace, (uint32_t)t, el)) * factor * pert;
        lg += gumbel_from_uniform(philox_uniform(e.seed, kStreamCatGumbel, (uint32_t)t, el));
        if (lg > best_v || (lg == best_v && c < best_c)) { best_v = lg; best_c = c; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, best_v, o);
      const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
      if (ov > best_v || (ov == best_v && oc < best_c)) { best_v = ov; best_c = oc; }
    }
    if (lane == 0) outz[k] = best_c;
  }
}

// ---------------------------------------------------------------------------
// suggest, one CTA (NT threads) per batch fly: the same arithmetic as eagle_suggest_block with the
// loops over the pool spread over the CTA (the one-warp-per-fly form is a ~2000-instruction latency
// chain; in the cooperative grid kernel there are more CTAs than flies).  Sums over the pool are
// formed per warp and combined in a fixed order.  Dynamic smem: eagle_suggest_cta_smem(e) bytes.
// ---------------------------------------------------------------------------
template <int NT>
__device__ __forceinline__ void eagle_suggest_cta(const EagleDev& e, int b, double* smem) {
  constexpr int NW = NT / 32;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int P = e.P, B = e.B, D = e.D, Dk = e.Dk;
  const int t = *e.iter;
  const int nb = P / B;
  const int i = (t % nb) * B + b;
  double* s_f = smem;                          // [P]
  double* s_x = s_f + P;                       // [D]
  double* s_part = s_x + D;                    // [NW][D + 2]  per-warp partial sums
  double* s_bc = s_part + NW * (D + 2);        // [4] broadcast scalars
  double* s_lg = s_bc + 4;                     // [64] categorical logits
  int32_t* s_z = reinterpret_cast<int32_t*>(s_lg + 64);   // [Dk]
  int* s_cnt = s_z + Dk + (Dk & 1);            // [2 * NW]
  for (int d = tid; d < D; d += NT) s_x[d] = e.pool[(size_t)i * D + d];
  for (int d = tid; d < Dk; d += NT) s_z[d] = e.pool_z[(size_t)i * Dk + d];
  __syncthreads();
  double* out = e.batch + (size_t)b * D;
  int32_t* outz = e.batch_z + (size_t)b * Dk;
  if (t < nb) {  // still initialising: return the pool features (projected)
    for (int d = tid; d < D; d += NT) out[d] = fmin(fmax(s_x[d], 0.0), 1.0);
    for (int d = tid; d < Dk; d += NT) outz[d] = s_z[d];
    __syncthreads();
    return;
  }
  const double ri = e.rewards[i];
  const double cexp = -e.cfg.visibility / (double)e.norm_dim * 10.0;
  int npull = 0, npush = 0;
  for (int j = tid; j < P; j += NT) {
    const double d2 = fly_distance(s_x, e.pool + (size_t)j * D, D, s_z, e.pool_z + (size_t)j * Dk, Dk);
    const double rj = e.rewards[j];
    const double dir = rj - ri;
    const double sd = (dir >= 0.0) ? e.cfg.gravity : -e.cfg.negative_gravity;
    const double f = sd * exp(cexp * d2) * (isfinite(rj) ? 1.0 : 0.0);
    s_f[j] = f;
    npull += (f > 0.0);
    npush += (f < 0.0);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    npull += __shfl_xor_sync(0xffffffffu, npull, o);
    npush += __shfl_xor_sync(0xffffffffu, npush, o);
  }
  if (lane == 0) { s_cnt[warp] = npull; s_cnt[NW + warp] = npush; }
  __syncthreads();
  npull = npush = 0;
  for (int w = 0; w < NW; ++w) { npull += s_cnt[w]; npush += s_cnt[NW + w]; }
  if (e.cfg.mutate_normalization_type == 1) {
    // RANDOM normalisation (see eagle_suggest_block)
    double s1 = 0.0, s2 = 0.0;
    for (int j = tid; j < P; j += NT) {
      const double pos = s_f[j] > 0.0 ? 1.0 : 0.0;
      s1 += philox_uniform(e.seed, kStreamPullRand, (uint32_t)t, (uint64_t)b * P + j) * pos;
      s2 += philox_uniform(e.seed, kStreamPushRand, (uint32_t)t, (uint64_t)b * P + j) * pos;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) { s_part[warp * (D + 2)] = s1; s_part[warp * (D + 2) + 1] = s2; }
    __syncthreads();
    s1 = s2 = 0.0;
    for (int w = 0; w < NW; ++w) { s1 += s_part[w * (D + 2)]; s2 += s_part[w * (D + 2) + 1]; }
    __syncthreads();
    for (int j = tid; j < P; j += NT) {
      const double f = s_f[j];
      const double pos = f > 0.0 ? 1.0 : 0.0;
      const double w1 = s1 > 0.0 ? philox_uniform(e.seed, kStreamPullRand, (uint32_t)t, (uint64_t)b * P + j) * pos / s1 : 0.0;
      const double w2 = s2 > 0.0 ? philox_uniform(e.seed, kStreamPushRand, (uint32_t)t, (uint64_t)b * P + j) * pos / s2 : 0.0;
      s_f[j] = e.cfg.normalization_scale * fmax(f, 0.0) * w1 + e.cfg.normalization_scale * fmin(f, 0.0) * w2;
    }
  } else {
    const double wpull = npull > 0 ? e.cfg.normalization_scale / (double)npull : 0.0;
    const double wpush = npush > 0 ? e.cfg.normalization_scale / (double)npush : 0.0;
    for (int j = tid; j < P; j += NT) {
      const double f = s_f[j];
      s_f[j] = f > 0.0 ? f * wpull : (f < 0.0 ? f * wpush : 0.0);
    }
  }
  __syncthreads();
  // ---- continuous features: warp w sums flies w, w + NW, ...; lane = dimension (and lane + 32) ----
  {
    double a0 = 0.0, a1 = 0.0, ss = 0.0;
    const int d0 = lane, d1 = lane + 32;
    for (int j = warp; j < P; j += NW) {
      const double sc = s_f[j];
      ss += sc;
      const double* pj = e.pool + (size_t)j * D;
      if (d0 < D) a0 = fma(sc, pj[d0], a0);
      if (d1 < D) a1 = fma(sc, pj[d1], a1);
    }
    if (d0 < D) s_part[warp * (D + 2) + d0] = a0;
    if (d1 < D) s_part[warp * (D + 2) + d1] = a1;
    if (lane == 0) s_part[warp * (D + 2) + D] = ss;
  }
  __syncthreads();
  const double pert = e.pert[i];
  double ssum = 0.0;
  for (int w = 0; w < NW; ++w) ssum += s_part[w * (D + 2) + D];
  for (int d = tid; d < D; d += NT) {
    double acc = 0.0;
    for (int w = 0; w < NW; ++w) acc += s_part[w * (D + 2) + d];
    const double u = philox_uniform(e.seed, kStreamPerturbSign, (uint32_t)t, (uint64_t)b * D + d);
    const double v = s_x[d] + (acc - s_x[d] * ssum) + (u >= 0.5 ? pert : -pert);
    out[d] = fmin(fmax(v, 0.0), 1.0);
  }
  // ---- categorical features: warp w takes categories w, w + NW, ...; lanes sum over the pool ----
  if (Dk > 0) {
    const double factor = D > 0 ? e.cfg.categorical_perturbation_factor : e.cfg.pure_categorical_perturbation_factor;
    const double log_same = log(e.cfg.prob_same_category_without_perturbation);
    for (int k = 0; k < Dk; ++k) {
      const int size = e.sizes[k];
      __syncthreads();
      if (size <= 1) {
        if (tid == 0) outz[k] = 0;
        continue;
      }
      const double log_diff = log((1.0 - e.cfg.prob_same_category_without_perturbation) / ((double)size - 1.0));
      for (int c = warp; c < size; c += NW) {
        double lg = 0.0;
        for (int j = lane; j < P; j += 32) lg += (e.pool_z[(size_t)j * Dk + k] == c) ? s_f[j] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lg += __shfl_xor_sync(0xffffffffu, lg, o);
        if (lane == 0) {
          lg += log_diff;
          if (c == s_z[k]) lg += -ssum + log_same - log_diff;
          const uint64_t el = ((uint64_t)b * Dk + k) * e.smax + c;
          lg += laplace_from_uniform(philox_uniform(e.seed, kStreamCatLaplace, (uint32_t)t, el)) * factor * pert;
          lg += gumbel_from_uniform(philox_uniform(e.seed, kStreamCatGumbel, (uint32_t)t, el));
          s_lg[c] = lg;
        }
      }
      __syncthreads();
      if (tid == 0) {
        double best_v = -INFINITY;
        int best_c = 0;
        for (int c = 0; c < size; ++c)
          if (s_lg[c] > best_v) { best_v = s_lg[c]; best_c = c; }
        outz[k] = best_c;
      }
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// update + trim + top-count bookkeeping: single CTA.  Dynamic smem: (B+count) doubles + flags.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool rank_better(double v, long long id, double bv, long long bid) {
  return (v > bv) || (v == bv && id < bid);
}

// The first 256 threads of the CTA run the update; NAMED = true synchronises only those (named barrier 1)
// so that the remaining warps of a larger CTA can wait at the next CTA-wide barrier.
template <bool NAMED>
__device__ __forceinline__ void eagle_update_block(const EagleDev& e, double* smem) {
  auto sync = [] { if (NAMED) asm volatile("bar.sync 1, 256;\n" ::: "memory"); else __syncthreads(); };
  __shared__ double sv[256];
  __shared__ long long si[256];
  __shared__ int sp[256];
  const int tid = threadIdx.x;
  const int P = e.P, B = e.B, D = e.D, Dk = e.Dk, count = e.count;
  const int t = *e.iter;
  const int nb = P / B;
  const int start = (t % nb) * B;
  // new best reward
  double m = -INFINITY;
  for (int b = tid; b < B; b += 256) m = fmax(m, e.batch_r[b]);
  sv[tid] = m;
  sync();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) sv[tid] = fmax(sv[tid], sv[tid + o]);
    sync();
  }
  const double new_best = fmax(*e.best_reward, sv[0]);
  sync();

  // ---- top-count merge of (batch U best) into tmp, then copy back ----
  double* cv = smem;                                        // [B+count] ranking values
  unsigned char* used = reinterpret_cast<unsigned char*>(cv + B + count);  // [B+count]
  for (int q = tid; q < B + count; q += 256) {
    double v = q < B ? e.batch_r[q] : e.best_r[q - B];
    cv[q] = isnan(v) ? -INFINITY : v;
    used[q] = 0;
  }
  sync();
  for (int c = 0; c < count; ++c) {
    double bv = -INFINITY;
    long long bid = LLONG_MAX;
    int bp = -1;
    for (int q = tid; q < B + count; q += 256) {
      if (used[q]) continue;
      long long id = q < B ? (long long)t * B + q : e.best_id[q - B];
      if (bp < 0 || rank_better(cv[q], id, bv, bid)) { bv = cv[q]; bid = id; bp = q; }
    }
    sv[tid] = bv; si[tid] = bid; sp[tid] = bp;
    sync();
    for (int o = 128; o > 0; o >>= 1) {
      if (tid < o && sp[tid + o] >= 0 &&
          (sp[tid] < 0 || rank_better(sv[tid + o], si[tid + o], sv[tid], si[tid]))) {
        sv[tid] = sv[tid + o]; si[tid] = si[tid + o]; sp[tid] = sp[tid + o];
      }
      sync();
    }
    const int q = sp[0];
    const long long qid = si[0];
    sync();
    if (q >= 0) {
      const double* src = q < B ? e.batch + (size_t)q * D : e.best_x + (size_t)(q - B) * D;
      const int32_t* srcz = q < B ? e.batch_z + (size_t)q * Dk : e.best_z + (size_t)(q - B) * Dk;
      for (int d = tid; d < D; d += 256) e.tmp_x[(size_t)c * D + d] = src[d];
      for (int d = tid; d < Dk; d += 256) e.tmp_z[(size_t)c * Dk + d] = srcz[d];
      if (tid == 0) {
        e.tmp_r[c] = q < B ? e.batch_r[q] : e.best_r[q - B];
        e.tmp_id[c] = qid;
        used[q] = 1;
      }
    }
    sync();
  }
  for (int q = tid; q < count * D; q += 256) e.best_x[q] = e.tmp_x[q];
  for (int q = tid; q < count * Dk; q += 256) e.best_z[q] = e.tmp_z[q];
  for (int c = tid; c < count; c += 256) { e.best_r[c] = e.tmp_r[c]; e.best_id[c] = e.tmp_id[c]; }

  // ---- pool update ----
  for (int b = tid; b < B; b += 256) {
    const int i = start + b;
    const double rb = e.batch_r[b];
    double pert = e.pert[i];
    if (t < nb) {
      for (int d = 0; d < D; ++d) e.pool[(size_t)i * D + d] = e.batch[(size_t)b * D + d];
      for (int d = 0; d < Dk; ++d) e.pool_z[(size_t)i * Dk + d] = e.batch_z[(size_t)b * Dk + d];
      e.rewards[i] = rb;
    } else {
      const double prev = e.rewards[i];
      const bool improve = rb > prev;
      double nr = improve ? rb : prev;
      if (!improve) pert *= e.cfg.penalize_factor;
      const bool trim = (pert < e.cfg.perturbation_lower_bound) && (nr != new_best);
      if (trim) {
        for (int d = 0; d < D; ++d)
          e.pool[(size_t)i * D + d] = philox_uniform(e.seed, kStreamTrim, (uint32_t)t, (uint64_t)b * D + d);
        for (int d = 0; d < Dk; ++d)
          e.pool_z[(size_t)i * Dk + d] = uniform_category(
              philox_uniform(e.seed, kStreamTrimCat, (uint32_t)t, (uint64_t)b * Dk + d), e.sizes[d]);
        pert = e.cfg.perturbation;
        nr = -INFINITY;
      } else if (improve) {
        for (int d = 0; d < D; ++d) e.pool[(size_t)i * D + d] = e.batch[(size_t)b * D + d];
        for (int d = 0; d < Dk; ++d) e.pool_z[(size_t)i * Dk + d] = e.batch_z[(size_t)b * Dk + d];
      }
      e.rewards[i] = nr;
      e.pert[i] = pert;
    }
  }
  sync();
  if (tid == 0) { *e.best_reward = new_best; *e.iter = t + 1; }
}

}  // namespace vzgp
