// Gradient of the GP negative log marginal likelihood w.r.t. the ARD hyper-parameters.
//
// Replaces the JAX autodiff of loss_with_aux (vizier/_src/jax/stochastic_process_model.py:
// 940-966, differentiated at vizier/_src/jax/optimizers/jaxopt_wrappers.py:149-151) by the
// closed form (SURVEY A.3):  G = K_y^-1 - alpha alpha^T,  dNLL/dp = 0.5 * sum_ij G_ij dK_ij/dp,
//   dK/d ls2_d = -E_ij * diff_ijd^2 / ls2_d^2,  dK/d sf2 = K/sf2,  dK_y/d sn2 = I,
//   E_ij = dk/d(d2) = -(5/6) sf2 (1+s) exp(-s).
#include "launchers.h"
#include "tiles.cuh"

namespace vzgp {

using G64 = GemmCfg<64, 64, 16, 4, 4>;

// One CTA per lower-triangular 64x64 tile (off-diagonal tiles count twice).  Writes
// partial[tile][0..dk) = sum G*E*neq_k, [dk..dk+dc) = sum G*E*diff_d^2, [dk+dc] = trace part of G,
// [dk+dc+1] = sum G*K_matern; with the linear_coef model (kp.use_linear) three more groups follow:
// [dk+dc+2 .. +dc) = sum G (x_id u_jd + x_jd u_id), then sum G sum_d u_id u_jd, then sum G sum_d (u_id + u_jd),
// u_id = x_id / l_d - coef*shift  (the pieces of dK_lin/d ls2_d, d/d slope, d/d shift).  WIDE (Dk > kMaxDk): the
// categorical features are staged kCatTile at a time (tiles.cuh), once for d2 and once for their gradient sums.
template <bool WIDE>
__global__ void __launch_bounds__(256) k_nll_grad_tiles(const double* __restrict__ X,
                                                        const int32_t* __restrict__ Z, int np,
                                                        int n_valid, KernelParams kp,
                                                        const double* __restrict__ Kinv, int ldk, int kc,
                                                        const double* __restrict__ alpha,
                                                        double* __restrict__ partial, int nb, int n_metrics,
                                                        int astride) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  extern __shared__ double smem[];
  constexpr int LD = 66;
  const int dc = kp.dc, dk = kp.dk, np_out = dc + dk + 2 + (kp.use_linear ? dc + 2 : 0);
  double* sa = smem;
  double* sb = sa + dc * LD;
  double* s_part = sb + dc * LD;                                   // [8 warps][np_out]
  int32_t* za = reinterpret_cast<int32_t*>(s_part + 8 * np_out);
  int32_t* zb = za + (WIDE ? kCatTile : dk) * LD;
  stage_rows_T(X, np, dc, bi * 64, 64, sa, LD);
  stage_rows_T(X, np, dc, bj * 64, 64, sb, LD);
  if (!WIDE && dk > 0) {
    stage_rows_T_i32(Z, np, dk, bi * 64, 64, za, LD);
    stage_rows_T_i32(Z, np, dk, bj * 64, 64, zb, LD);
  }
  __syncthreads();
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16, warp = tid / 32, lane = tid % 32;
  double d2[4][4], unused[4][4];
  tile_d2<G64, 4, 4, false, !WIDE>(sa, LD, sb, LD, za, LD, zb, LD, kp, nullptr, ty, tx, d2, unused);
  if (WIDE)
    for_cat_tiles(Z, np, bi * 64, 64, Z, np, bj * 64, 64, dk, za, LD, zb, LD, [&](int k0, int kt) {
      tile_hamming<G64, 4, 4>(za, LD, zb, LD, kp.inv_ls2_k_wide + k0, kt, ty, tx, d2);
    });
  double ge[4][4], gg[4][4];
  double sum_gk = 0.0, sum_tr = 0.0;
  const double wgt = (bi == bj) ? 1.0 : 2.0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gi = bi * 64 + G64::row_of(ty, i), gj = bj * 64 + G64::col_of(tx, j);
      double g = 0.0, kv = 0.0, ev = 0.0;
      if (gi < n_valid && gj < n_valid) {
        double kinv = 0.0;   // planes of k_lauum that meet k >= 64*bi, ascending
        for (int z = (bi * 64) / kc; z < kLauumSplit && z * kc < np; ++z)
          kinv += Kinv[((size_t)z * np + gi) * ldk + gj];
        double aa = 0.0;   // independent multi-task GP: G = M K_y^-1 - sum_m alpha_m alpha_m^T
        for (int m = 0; m < n_metrics; ++m) aa = fma(alpha[(size_t)m * astride + gi], alpha[(size_t)m * astride + gj], aa);
        g = wgt * (n_metrics * kinv - aa);
        matern52_with_grad(d2[i][j], kp.sf2, kv, ev);
        if (gi == gj) sum_tr += g;
      }
      ge[i][j] = g * ev;
      gg[i][j] = g;
      sum_gk = fma(g, kv, sum_gk);
    }
  auto warp_store = [&](double v, int slot) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) s_part[warp * np_out + slot] = v;
  };
  auto cat_sums = [&](int k0, int kt) {
    for (int k = 0; k < kt; ++k) {
      double t = 0.0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int av = za[k * LD + G64::row_of(ty, i)];
#pragma unroll
        for (int j = 0; j < 4; ++j) t += (av != zb[k * LD + G64::col_of(tx, j)]) ? ge[i][j] : 0.0;
      }
      warp_store(t, k0 + k);
    }
  };
  if (WIDE) for_cat_tiles(Z, np, bi * 64, 64, Z, np, bj * 64, 64, dk, za, LD, zb, LD, cat_sums);
  else cat_sums(0, dk);
  for (int d = 0; d < dc; ++d) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const double av = sa[d * LD + G64::row_of(ty, i)];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double diff = av - sb[d * LD + G64::col_of(tx, j)];
        t = fma(ge[i][j], diff * diff, t);
      }
    }
    warp_store(t, dk + d);
  }
  warp_store(sum_tr, dk + dc);
  warp_store(sum_gk, dk + dc + 1);
  if (kp.use_linear) {
    double q = 0.0, hs = 0.0;
    for (int d = 0; d < dc; ++d) {
      const double w = kp.inv_ls_c[d];
      double xi[4], ui[4], xj[4], uj[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { xi[i] = sa[d * LD + G64::row_of(ty, i)]; ui[i] = fma(xi[i], w, -kp.lin_b); }
#pragma unroll
      for (int j = 0; j < 4; ++j) { xj[j] = sb[d * LD + G64::col_of(tx, j)]; uj[j] = fma(xj[j], w, -kp.lin_b); }
      double t = 0.0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          t = fma(gg[i][j], fma(xi[i], uj[j], xj[j] * ui[i]), t);
          q = fma(gg[i][j], ui[i] * uj[j], q);
          hs = fma(gg[i][j], ui[i] + uj[j], hs);
        }
      warp_store(t, dk + dc + 2 + d);
    }
    warp_store(q, dk + dc + 2 + dc);
    warp_store(hs, dk + dc + 2 + dc + 1);
  }
  __syncthreads();
  // tile index in row-major lower-triangular enumeration
  const int tile = bi * (bi + 1) / 2 + bj;
  auto slot_sum = [&](int q) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_part[w * np_out + q];
    partial[(size_t)tile * np_out + q] = s;
  };
  if (WIDE) for (int q = tid; q < np_out; q += 256) slot_sum(q);   // np_out > 256 only here
  else if (tid < np_out) slot_sum(tid);
}

// out[q] = sum over tiles (fixed order) of partial[tile][q].
__global__ void k_reduce_partials(const double* __restrict__ partial, int ntiles, int nq,
                                  double* __restrict__ out) {
  __shared__ double red[32];
  const int q = blockIdx.x;
  double s = 0.0;
  for (int t = threadIdx.x; t < ntiles; t += blockDim.x) s += partial[(size_t)t * nq + q];
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[q] = s;
}

static_assert(KernelArgs<decltype(&k_nll_grad_tiles<false>)>::count == kNllGradTilesArgs &&
              std::is_same<KernelArgs<decltype(&k_nll_grad_tiles<false>)>::arg<kNllGradTilesKpArg>, KernelParams>::value,
              "k_nll_grad_tiles signature changed: update kNllGradTiles*Arg in launchers.h");
const void* nll_grad_tiles_func(bool wide) {
  return wide ? reinterpret_cast<const void*>(&k_nll_grad_tiles<true>) : reinterpret_cast<const void*>(&k_nll_grad_tiles<false>);
}

int launch_nll_grad_tiles(vzgp_handle* h, const double* X, const int32_t* Z, int np, int n_valid,
                          const KernelParams& kp, const double* Kinv, int ldk, const double* alpha,
                          double* partial, double* out, int plane_rows, int n_metrics) {
  const int nb = np / 64, nq = kp.dc + kp.dk + 2 + (kp.use_linear ? kp.dc + 2 : 0), ntiles = nb * (nb + 1) / 2;
  const bool wide = kp.dk > kMaxDk;
  size_t sm = sizeof(double) * (kp.dc * 2 * 66 + 8 * nq) + sizeof(int32_t) * (wide ? kCatTile : kp.dk) * 2 * 66;
  const auto kfn = wide ? k_nll_grad_tiles<true> : k_nll_grad_tiles<false>;
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  kfn<<<dim3(nb, nb), 256, sm, h->stream>>>(X, Z, np, n_valid, kp, Kinv, ldk, plane_rows > 0 ? plane_rows : lauum_plane_rows(np), alpha,
                                                         partial, nb, n_metrics, np);
  VZ_CHECK_LAUNCH();
  k_reduce_partials<<<nq, 256, 0, h->stream>>>(partial, ntiles, nq, out);
  VZ_CHECK_LAUNCH();
  h->launches += 2;
  return 0;
}

}  // namespace vzgp
