// The stages of one NLL + gradient evaluation of a small study (N <= 64) in one CTA of 256 threads, shared by
// k_nll_grad_small (nll_small.cu: one evaluation per launch) and k_ard_adam_small (ard_adam.cu: every Adam epoch of
// one ARD restart per CTA):
//   nll_small_stage:  features (transposed), categorical features and labels into shared memory, once per launch;
//   nll_small_eval:   K_y build -> Cholesky + inverse with the jitter retry loop (tuned_gp_models.py:272-280) ->
//                     alpha (+ one refinement step) -> K_y^-1 = L^-T L^-1 -> log-det, quadratic form ->
//                     gradient contraction  sum_ij (K_y^-1 - alpha alpha^T)_ij dK_ij/dtheta  (SURVEY A.3).
// Same arithmetic and conventions as the general path (padded rows are identity rows, the shift goes on every
// diagonal entry, reductions in a fixed order).
#pragma once

#include "device.cuh"
#include "potf2.cuh"
#include "tiles.cuh"

namespace vzgp {

constexpr int kSmallLD = 66;

__device__ __forceinline__ double small_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// Shared-memory layout of one evaluation (bytes: nll_small_smem_bytes in nll_small.cu).
struct SmallNllSmem {
  double *ky, *d2m, *a, *x, *t, *xt, *yv, *wv, *al, *rv, *tv, *rd, *s_part;
  int32_t* zt;
  __device__ __forceinline__ SmallNllSmem(double* smem, int dc, int nq) {
    ky = smem;                 // [64][66] K_y (unshifted), full symmetric
    d2m = ky + 64 * kSmallLD;  // [64][66] squared scaled distances
    a = d2m + 64 * kSmallLD;   // [64][66] factor
    x = a + 64 * kSmallLD;     // [64][66] inverse factor, later K_y^-1
    t = x + 64 * kSmallLD;     // [32][34]
    xt = t + 32 * 34;          // [dc][66] features, transposed
    yv = xt + dc * kSmallLD;   // [64]
    wv = yv + 64;              // [64] L^-1 y
    al = wv + 64;              // [64] alpha
    rv = al + 64;              // [64] residual / temporaries
    tv = rv + 64;              // [64]
    rd = tv + 64;              // [64]
    s_part = rd + 64;          // [8][nq]
    zt = reinterpret_cast<int32_t*>(s_part + 8 * nq);   // [dk][66]  (WIDE: [kCatTile][66])
  }
  // first double past the layout (8-byte aligned: the categorical block holds an even number of int32)
  __device__ __forceinline__ double* end(int zk) const { return reinterpret_cast<double*>(zt + zk * kSmallLD); }
};

// Features and labels into shared memory (the caller synchronises before nll_small_eval).
template <bool WIDE>
__device__ __forceinline__ void nll_small_stage(const double* __restrict__ X, const int32_t* __restrict__ Z,
                                                const double* __restrict__ y, int N, int n_valid, int dc, int dk,
                                                double* smem) {
  const SmallNllSmem s(smem, dc, dc + dk + 2);
  const int tid = threadIdx.x;
  for (int e = tid; e < 64 * dc; e += 256) {
    const int i = e / dc, d = e - i * dc;
    s.xt[d * kSmallLD + i] = i < N ? X[(size_t)i * dc + d] : 0.0;
  }
  for (int e = tid; !WIDE && e < 64 * dk; e += 256) {
    const int i = e / dk, k = e - i * dk;
    s.zt[k * kSmallLD + i] = i < N ? Z[(size_t)i * dk + k] : -1;
  }
  if (tid < 64) s.yv[tid] = tid < n_valid ? y[tid] : 0.0;
}

// One evaluation on the staged data.  kp: dc, dk, sf2, inv_ls2_c, inv_ls2_k (Dk <= kMaxDk); wide_w(k): the inverse
// squared length scale of categorical feature k (WIDE only).
// out: [0] = sum_i log L_ii (i < N), [1] = 0.5 * |L^-1 y|^2, [2] = shift used, [3] = retries
//      (max_iters + 1 = never succeeded), [4 .. 4 + nq) = raw gradient sums in the order
//      categorical (G E neq_k), continuous (G E diff_d^2), trace(G), sum(G K).
// WIDE (Dk > kMaxDk): the categorical features are staged kCatTile at a time (tiles.cuh), and d2 takes the Hamming
// term tile by tile in ascending feature order, the order of the one-pass sum.
// s_bad: a shared int of the caller's (the pivot flag of the factorisation).
// The last writes to `out` are not followed by a barrier.
template <bool WIDE, class WideW>
__device__ __forceinline__ void nll_small_eval(const int32_t* __restrict__ Z, int N, int n_valid, const KernelParams& kp,
                                               WideW wide_w, double sn2, double jitter0, int max_iters,
                                               double* smem, int* s_bad, double* out) {
  const int dc = kp.dc, dk = kp.dk, nq = dc + dk + 2;
  const SmallNllSmem s(smem, dc, nq);
  double* const ky = s.ky;
  double* const d2m = s.d2m;
  double* const a = s.a;
  double* const x = s.x;
  double* const xt = s.xt;
  double* const yv = s.yv;
  double* const wv = s.wv;
  double* const al = s.al;
  double* const rv = s.rv;
  double* const tv = s.tv;
  double* const s_part = s.s_part;
  int32_t* const zt = s.zt;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- K_y and d2 (thread -> row i = e / 64... 16 entries each, symmetric computed twice) ----
  for (int e = tid; e < 64 * 64; e += 256) {
    const int i = e >> 6, j = e & 63;
    double v2 = 0.0;
    for (int d = 0; d < dc; ++d) {
      const double df = xt[d * kSmallLD + i] - xt[d * kSmallLD + j];
      v2 = fma(df * df, kp.inv_ls2_c[d], v2);
    }
    if (!WIDE)
      for (int k = 0; k < dk; ++k) v2 += (zt[k * kSmallLD + i] != zt[k * kSmallLD + j]) ? kp.inv_ls2_k[k] : 0.0;
    d2m[i * kSmallLD + j] = v2;
    if (WIDE) continue;
    double v;
    if (i >= n_valid || j >= n_valid) v = (i == j) ? 1.0 : 0.0;
    else { v = matern52(v2, kp.sf2); if (i == j) v += sn2; }
    ky[i * kSmallLD + j] = v;
  }
  if (WIDE) {
    for_cat_tiles(Z, N, 0, 64, nullptr, 0, 0, 0, dk, zt, kSmallLD, nullptr, 0, [&](int k0, int kt) {
      for (int e = tid; e < 64 * 64; e += 256) {
        const int i = e >> 6, j = e & 63;
        double v2 = d2m[i * kSmallLD + j];
        for (int k = 0; k < kt; ++k) v2 += (zt[k * kSmallLD + i] != zt[k * kSmallLD + j]) ? wide_w(k0 + k) : 0.0;
        d2m[i * kSmallLD + j] = v2;
      }
    });
    for (int e = tid; e < 64 * 64; e += 256) {
      const int i = e >> 6, j = e & 63;
      double v;
      if (i >= n_valid || j >= n_valid) v = (i == j) ? 1.0 : 0.0;
      else { v = matern52(d2m[i * kSmallLD + j], kp.sf2); if (i == j) v += sn2; }
      ky[i * kSmallLD + j] = v;
    }
  }
  __syncthreads();
  // ---- Cholesky with retry ----
  double shift = 0.0;
  int attempt = 0;
  for (;;) {
    if (tid == 0) *s_bad = 0;
    for (int e = tid; e < 64 * 64; e += 256) {
      const int i = e >> 6, j = e & 63;
      const bool upper_blk = (j >> 4) > (i >> 4);
      a[i * kSmallLD + j] = upper_blk ? 0.0 : ky[i * kSmallLD + j] + ((i == j) ? shift : 0.0);
      x[i * kSmallLD + j] = 0.0;
    }
    __syncthreads();
    potf2_inv_64(a, x, s.t, s.rd, s_bad);
    __syncthreads();
    const int bad = *s_bad;
    __syncthreads();
    if (!bad) break;
    if (attempt >= max_iters) { attempt = max_iters + 1; break; }
    shift = (shift == 0.0) ? jitter0 : shift * 10.0;
    ++attempt;
  }
  // ---- alpha = L^-T (L^-1 y), one refinement step against K_y + shift I ----
  auto lower_mv = [&](const double* v, double* o) {       // o = Linv v
    if (tid < 64) {
      double acc = 0.0;
      for (int k = 0; k <= tid; ++k) acc = fma(x[tid * kSmallLD + k], v[k], acc);
      o[tid] = acc;
    }
    __syncthreads();
  };
  auto lower_tmv = [&](const double* v, double* o) {      // o = Linv^T v
    if (tid < 64) {
      double acc = 0.0;
      for (int k = tid; k < 64; ++k) acc = fma(x[k * kSmallLD + tid], v[k], acc);
      o[tid] = acc;
    }
    __syncthreads();
  };
  lower_mv(yv, wv);
  lower_tmv(wv, al);
  if (tid < 64) {
    double acc = yv[tid];
    for (int k = 0; k < 64; ++k) acc = fma(-ky[tid * kSmallLD + k], al[k], acc);
    rv[tid] = acc - shift * al[tid];
  }
  __syncthreads();
  lower_mv(rv, tv);
  lower_tmv(tv, rv);
  if (tid < 64) al[tid] += rv[tid];
  // ---- log-det and quadratic form ----
  if (warp == 0) {
    double lg = 0.0, q = 0.0;
    // log-det over all N rows: a masked (identity) row adds log(1 + shift) once the jitter fires (k_logdet_quad)
    for (int i = lane; i < N; i += 32) {
      lg += log(a[i * kSmallLD + i]);
      if (i < n_valid) q = fma(wv[i], wv[i], q);
    }
    lg = small_warp_sum(lg); q = small_warp_sum(q);
    if (lane == 0) { out[0] = lg; out[1] = 0.5 * q; out[2] = shift; out[3] = (double)attempt; }
  }
  __syncthreads();
  // ---- K_y^-1 = Linv^T Linv into a (full symmetric) ----
  for (int e = tid; e < 64 * 64; e += 256) {
    const int i = e >> 6, j = e & 63;
    const int k0 = i > j ? i : j;
    double acc = 0.0;
    for (int k = k0; k < 64; ++k) acc = fma(x[k * kSmallLD + i], x[k * kSmallLD + j], acc);
    a[i * kSmallLD + j] = acc;   // the factor itself is no longer needed
  }
  __syncthreads();
  // ---- gradient sums: g = Kinv - alpha alpha^T over valid pairs ----
  double ge[16];
  double sum_tr = 0.0, sum_gk = 0.0;
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int e = tid + 256 * u, i = e >> 6, j = e & 63;
    double g = 0.0, kv = 0.0, ev = 0.0;
    if (i < n_valid && j < n_valid) {
      g = a[i * kSmallLD + j] - al[i] * al[j];
      matern52_with_grad(d2m[i * kSmallLD + j], kp.sf2, kv, ev);
      if (i == j) sum_tr += g;
    }
    ge[u] = g * ev;
    sum_gk = fma(g, kv, sum_gk);
  }
  auto warp_store = [&](double v, int slot) {
    v = small_warp_sum(v);
    if (lane == 0) s_part[warp * nq + slot] = v;
  };
  auto cat_sums = [&](int k0, int kt) {
    for (int k = 0; k < kt; ++k) {
      double acc = 0.0;
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const int e = tid + 256 * u, i = e >> 6, j = e & 63;
        acc += (zt[k * kSmallLD + i] != zt[k * kSmallLD + j]) ? ge[u] : 0.0;
      }
      warp_store(acc, k0 + k);
    }
  };
  if (WIDE) for_cat_tiles(Z, N, 0, 64, nullptr, 0, 0, 0, dk, zt, kSmallLD, nullptr, 0, cat_sums);
  else cat_sums(0, dk);
  for (int d = 0; d < dc; ++d) {
    double acc = 0.0;
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int e = tid + 256 * u, i = e >> 6, j = e & 63;
      const double df = xt[d * kSmallLD + i] - xt[d * kSmallLD + j];
      acc = fma(ge[u], df * df, acc);
    }
    warp_store(acc, dk + d);
  }
  warp_store(sum_tr, dk + dc);
  warp_store(sum_gk, dk + dc + 1);
  __syncthreads();
  auto slot_sum = [&](int q) {
    double acc = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) acc += s_part[w * nq + q];
    out[4 + q] = acc;
  };
  if (WIDE) for (int q = tid; q < nq; q += 256) slot_sum(q);   // nq > 256 only here
  else if (tid < nq) slot_sum(tid);
}

}  // namespace vzgp
