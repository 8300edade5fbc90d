// NLL + gradient for small studies (N <= 64) in ONE kernel launch.
//
// The ARD loop (jaxopt_wrappers.py:108-199 driving stochastic_process_model.py:940-966) evaluates the
// loss a few hundred times per suggest().  For N <= 64 the general path is ~16 tiny launches and two
// host round trips per evaluation; here one CTA keeps the whole model in shared memory:
//   K_y build -> Cholesky + inverse with the jitter retry loop (tuned_gp_models.py:272-280) ->
//   alpha (+ one refinement step) -> K_y^-1 = L^-T L^-1 -> log-det, quadratic form ->
//   gradient contraction  sum_ij (K_y^-1 - alpha alpha^T)_ij dK_ij/dtheta  (SURVEY A.3).
// Same arithmetic and conventions as the general path (padded rows are identity rows, the shift goes on
// every diagonal entry, reductions in a fixed order); the host finishes with the regularisers.
#include "launchers.h"
#include "device.cuh"
#include "potf2.cuh"
#include "tiles.cuh"

namespace vzgp {

namespace {
constexpr int kLD = 66;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
}  // namespace

// out: [0] = sum_i log L_ii (i < N), [1] = 0.5 * |L^-1 y|^2, [2] = shift used, [3] = retries
//      (max_iters + 1 = never succeeded), [4 .. 4 + nq) = raw gradient sums in the order
//      categorical (G E neq_k), continuous (G E diff_d^2), trace(G), sum(G K).
// WIDE (Dk > kMaxDk): the categorical features are staged kCatTile at a time (tiles.cuh), and d2 takes the Hamming
// term tile by tile in ascending feature order, the order of the one-pass sum.  Without a minimum of one CTA per SM
// ptxas holds the wide form to 64 registers and spills.
template <bool WIDE>
__global__ void __launch_bounds__(256, WIDE ? 1 : 0) k_nll_grad_small(const double* __restrict__ X, const int32_t* __restrict__ Z,
                                                        const double* __restrict__ y, int N, int n_valid,
                                                        KernelParams kp, double sn2, double jitter0, int max_iters,
                                                        double* __restrict__ out) {
  extern __shared__ double smem[];
  const int dc = kp.dc, dk = kp.dk, nq = dc + dk + 2;
  double* ky = smem;                 // [64][66] K_y (unshifted), full symmetric
  double* d2m = ky + 64 * kLD;       // [64][66] squared scaled distances
  double* a = d2m + 64 * kLD;        // [64][66] factor
  double* x = a + 64 * kLD;          // [64][66] inverse factor, later K_y^-1
  double* t = x + 64 * kLD;          // [32][34]
  double* xt = t + 32 * 34;          // [dc][66] features, transposed
  double* yv = xt + dc * kLD;        // [64]
  double* wv = yv + 64;              // [64] L^-1 y
  double* al = wv + 64;              // [64] alpha
  double* rv = al + 64;              // [64] residual / temporaries
  double* tv = rv + 64;              // [64]
  double* rd = tv + 64;              // [64]
  double* s_part = rd + 64;          // [8][nq]
  int32_t* zt = reinterpret_cast<int32_t*>(s_part + 8 * nq);   // [dk][66]  (WIDE: [kCatTile][66])
  __shared__ int s_bad;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int e = tid; e < 64 * dc; e += 256) {
    const int i = e / dc, d = e - i * dc;
    xt[d * kLD + i] = i < N ? X[(size_t)i * dc + d] : 0.0;
  }
  for (int e = tid; !WIDE && e < 64 * dk; e += 256) {
    const int i = e / dk, k = e - i * dk;
    zt[k * kLD + i] = i < N ? Z[(size_t)i * dk + k] : -1;
  }
  if (tid < 64) yv[tid] = tid < n_valid ? y[tid] : 0.0;
  __syncthreads();
  // ---- K_y and d2 (thread -> row i = e / 64... 16 entries each, symmetric computed twice) ----
  for (int e = tid; e < 64 * 64; e += 256) {
    const int i = e >> 6, j = e & 63;
    double s = 0.0;
    for (int d = 0; d < dc; ++d) {
      const double df = xt[d * kLD + i] - xt[d * kLD + j];
      s = fma(df * df, kp.inv_ls2_c[d], s);
    }
    if (!WIDE)
      for (int k = 0; k < dk; ++k) s += (zt[k * kLD + i] != zt[k * kLD + j]) ? kp.inv_ls2_k[k] : 0.0;
    d2m[i * kLD + j] = s;
    if (WIDE) continue;
    double v;
    if (i >= n_valid || j >= n_valid) v = (i == j) ? 1.0 : 0.0;
    else { v = matern52(s, kp.sf2); if (i == j) v += sn2; }
    ky[i * kLD + j] = v;
  }
  if (WIDE) {
    for_cat_tiles(Z, N, 0, 64, nullptr, 0, 0, 0, dk, zt, kLD, nullptr, 0, [&](int k0, int kt) {
      for (int e = tid; e < 64 * 64; e += 256) {
        const int i = e >> 6, j = e & 63;
        double s = d2m[i * kLD + j];
        for (int k = 0; k < kt; ++k) s += (zt[k * kLD + i] != zt[k * kLD + j]) ? __ldg(kp.inv_ls2_k_wide + k0 + k) : 0.0;
        d2m[i * kLD + j] = s;
      }
    });
    for (int e = tid; e < 64 * 64; e += 256) {
      const int i = e >> 6, j = e & 63;
      double v;
      if (i >= n_valid || j >= n_valid) v = (i == j) ? 1.0 : 0.0;
      else { v = matern52(d2m[i * kLD + j], kp.sf2); if (i == j) v += sn2; }
      ky[i * kLD + j] = v;
    }
  }
  __syncthreads();
  // ---- Cholesky with retry ----
  double shift = 0.0;
  int attempt = 0;
  for (;;) {
    if (tid == 0) s_bad = 0;
    for (int e = tid; e < 64 * 64; e += 256) {
      const int i = e >> 6, j = e & 63;
      const bool upper_blk = (j >> 4) > (i >> 4);
      a[i * kLD + j] = upper_blk ? 0.0 : ky[i * kLD + j] + ((i == j) ? shift : 0.0);
      x[i * kLD + j] = 0.0;
    }
    __syncthreads();
    potf2_inv_64(a, x, t, rd, &s_bad);
    __syncthreads();
    const int bad = s_bad;
    __syncthreads();
    if (!bad) break;
    if (attempt >= max_iters) { attempt = max_iters + 1; break; }
    shift = (shift == 0.0) ? jitter0 : shift * 10.0;
    ++attempt;
  }
  // ---- alpha = L^-T (L^-1 y), one refinement step against K_y + shift I ----
  auto lower_mv = [&](const double* v, double* o) {       // o = Linv v
    if (tid < 64) {
      double s = 0.0;
      for (int k = 0; k <= tid; ++k) s = fma(x[tid * kLD + k], v[k], s);
      o[tid] = s;
    }
    __syncthreads();
  };
  auto lower_tmv = [&](const double* v, double* o) {      // o = Linv^T v
    if (tid < 64) {
      double s = 0.0;
      for (int k = tid; k < 64; ++k) s = fma(x[k * kLD + tid], v[k], s);
      o[tid] = s;
    }
    __syncthreads();
  };
  lower_mv(yv, wv);
  lower_tmv(wv, al);
  if (tid < 64) {
    double s = yv[tid];
    for (int k = 0; k < 64; ++k) s = fma(-ky[tid * kLD + k], al[k], s);
    rv[tid] = s - shift * al[tid];
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
      lg += log(a[i * kLD + i]);
      if (i < n_valid) q = fma(wv[i], wv[i], q);
    }
    lg = warp_sum(lg); q = warp_sum(q);
    if (lane == 0) { out[0] = lg; out[1] = 0.5 * q; out[2] = shift; out[3] = (double)attempt; }
  }
  __syncthreads();
  // ---- K_y^-1 = Linv^T Linv into a (full symmetric) ----
  for (int e = tid; e < 64 * 64; e += 256) {
    const int i = e >> 6, j = e & 63;
    const int k0 = i > j ? i : j;
    double s = 0.0;
    for (int k = k0; k < 64; ++k) s = fma(x[k * kLD + i], x[k * kLD + j], s);
    a[i * kLD + j] = s;   // the factor itself is no longer needed
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
      g = a[i * kLD + j] - al[i] * al[j];
      matern52_with_grad(d2m[i * kLD + j], kp.sf2, kv, ev);
      if (i == j) sum_tr += g;
    }
    ge[u] = g * ev;
    sum_gk = fma(g, kv, sum_gk);
  }
  auto warp_store = [&](double v, int slot) {
    v = warp_sum(v);
    if (lane == 0) s_part[warp * nq + slot] = v;
  };
  auto cat_sums = [&](int k0, int kt) {
    for (int k = 0; k < kt; ++k) {
      double s = 0.0;
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const int e = tid + 256 * u, i = e >> 6, j = e & 63;
        s += (zt[k * kLD + i] != zt[k * kLD + j]) ? ge[u] : 0.0;
      }
      warp_store(s, k0 + k);
    }
  };
  if (WIDE) for_cat_tiles(Z, N, 0, 64, nullptr, 0, 0, 0, dk, zt, kLD, nullptr, 0, cat_sums);
  else cat_sums(0, dk);
  for (int d = 0; d < dc; ++d) {
    double s = 0.0;
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int e = tid + 256 * u, i = e >> 6, j = e & 63;
      const double df = xt[d * kLD + i] - xt[d * kLD + j];
      s = fma(ge[u], df * df, s);
    }
    warp_store(s, dk + d);
  }
  warp_store(sum_tr, dk + dc);
  warp_store(sum_gk, dk + dc + 1);
  __syncthreads();
  auto slot_sum = [&](int q) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_part[w * nq + q];
    out[4 + q] = s;
  };
  if (WIDE) for (int q = tid; q < nq; q += 256) slot_sum(q);   // nq > 256 only here
  else if (tid < nq) slot_sum(tid);
}

size_t nll_small_smem_bytes(int dc, int dk) {
  const int nq = dc + dk + 2;
  const int zk = dk > kMaxDk ? kCatTile : dk;
  return sizeof(double) * (4 * 64 * kLD + 32 * 34 + (size_t)dc * kLD + 6 * 64 + 8 * nq) + sizeof(int32_t) * (size_t)zk * kLD;
}

int launch_nll_grad_small(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int n_valid,
                          const KernelParams& kp, double sn2, double jitter0, int max_iters, double* out) {
  const size_t sm = nll_small_smem_bytes(kp.dc, kp.dk);
  const auto kfn = kp.dk > kMaxDk ? k_nll_grad_small<true> : k_nll_grad_small<false>;
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  kfn<<<1, 256, sm, h->stream>>>(X, Z, y, N, n_valid, kp, sn2, jitter0, max_iters, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
