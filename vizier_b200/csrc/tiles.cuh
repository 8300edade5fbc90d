// Pairwise scaled-squared-distance tiles (the front half of every Matern kernel here).
#pragma once

#include "device.cuh"

namespace vzgp {

// Stages `rows` feature rows [row0, row0+rows) of X ([nrows x dc] row-major) into shared
// memory transposed: s[d*lds + r].  Rows >= nrows are filled with zeros.
__device__ __forceinline__ void stage_rows_T(const double* __restrict__ X, int nrows, int dc,
                                             int row0, int rows, double* s, int lds) {
  const int total = rows * dc;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    int r = e / dc, d = e - r * dc;
    int gr = row0 + r;
    s[d * lds + r] = gr < nrows ? __ldg(X + (size_t)gr * dc + d) : 0.0;
  }
}

__device__ __forceinline__ void stage_rows_T_i32(const int32_t* __restrict__ Z, int nrows, int dk,
                                                 int row0, int rows, int32_t* s, int lds,
                                                 int nthreads = 0) {
  const int total = rows * dk;
  const int stride = nthreads > 0 ? nthreads : (int)blockDim.x;
  for (int e = threadIdx.x; e < total; e += stride) {
    int r = e / dk, d = e - r * dk;
    int gr = row0 + r;
    s[d * lds + r] = gr < nrows ? __ldg(Z + (size_t)gr * dk + d) : -1;
  }
}

// d2[i][j] = sum_d (a_i[d]-b_j[d])^2 * inv_ls2[d]  (+ Hamming term), a/b staged by
// stage_rows_T.  The difference is formed before scaling so that it is exact for
// inputs in [0,1] (DESIGN.md, "accuracy of d2").  If WITH_LINF, also tracks
// linf[i][j] = max_{d in mask} |a_i[d]-b_j[d]| (trust region, acquisitions.py:779-820).
// CAT = false leaves out the categorical term (models past kMaxDk add it with tile_hamming, tile by tile).
template <typename Cfg, int TTM, int TTN, bool WITH_LINF, bool CAT = true>
__device__ __forceinline__ void tile_d2(const double* sa, int lda, const double* sb, int ldb,
                                        const int32_t* za, int ldza, const int32_t* zb, int ldzb,
                                        const KernelParams& kp, const uint8_t* tr_mask_smem,
                                        int ty, int tx, double (&d2)[TTM][TTN],
                                        double (&linf)[TTM][TTN]) {
#pragma unroll
  for (int i = 0; i < TTM; ++i)
#pragma unroll
    for (int j = 0; j < TTN; ++j) {
      d2[i][j] = 0.0;
      if (WITH_LINF) linf[i][j] = 0.0;
    }
  for (int d = 0; d < kp.dc; ++d) {
    double a[TTM], b[TTN];
#pragma unroll
    for (int i = 0; i < TTM; i += 2) {
      double2 t = *reinterpret_cast<const double2*>(sa + d * lda + Cfg::row_of(ty, i));
      a[i] = t.x; a[i + 1] = t.y;
    }
#pragma unroll
    for (int j = 0; j < TTN; j += 2) {
      double2 t = *reinterpret_cast<const double2*>(sb + d * ldb + Cfg::col_of(tx, j));
      b[j] = t.x; b[j + 1] = t.y;
    }
    const double w = kp.inv_ls2_c[d];
    const bool in_tr = WITH_LINF ? (tr_mask_smem[d] != 0) : false;
#pragma unroll
    for (int i = 0; i < TTM; ++i)
#pragma unroll
      for (int j = 0; j < TTN; ++j) {
        double diff = a[i] - b[j];
        d2[i][j] = fma(diff * diff, w, d2[i][j]);
        if (WITH_LINF && in_tr) linf[i][j] = fmax(linf[i][j], fabs(diff));
      }
  }
  if (!CAT) return;
  for (int k = 0; k < kp.dk; ++k) {
    const double w = kp.inv_ls2_k[k];
#pragma unroll
    for (int i = 0; i < TTM; ++i) {
      int av = za[k * ldza + Cfg::row_of(ty, i)];
#pragma unroll
      for (int j = 0; j < TTN; ++j) {
        int bv = zb[k * ldzb + Cfg::col_of(tx, j)];
        d2[i][j] += (av != bv) ? w : 0.0;
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Models with more than kMaxDk categorical features.  Their inverse length scales are a device array
// (kp.inv_ls2_k_wide), and the kernels stage the features kCatTile at a time, so shared memory does not grow with
// Dk.  The Hamming term is summed tile by tile in ascending feature order, the order of tile_d2's categorical loop.
// ---------------------------------------------------------------------------
// s[k * lds + r] = Z[row0 + r][k0 + k] for k < kt, r < rows (Z is [nrows x dk]); rows >= nrows read -1.
__device__ __forceinline__ void stage_cat_tile_T(const int32_t* __restrict__ Z, int nrows, int dk, int k0, int kt,
                                                 int row0, int rows, int32_t* s, int lds) {
  const int total = rows * kt;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int r = e / kt, k = e - r * kt;
    const int gr = row0 + r;
    s[k * lds + r] = gr < nrows ? __ldg(Z + (size_t)gr * dk + k0 + k) : -1;
  }
}

// Calls f(k0, kt) once per tile of categorical features [k0, k0 + kt), after rows [rowa, rowa + rows_a) of Za and
// [rowb, rowb + rows_b) of Zb are staged into za / zb ([kCatTile][ld]).  Every thread of the block calls it; it
// begins with a barrier (the previous tile's readers) and leaves the last tile staged.
template <class F>
__device__ __forceinline__ void for_cat_tiles(const int32_t* __restrict__ Za, int na, int rowa, int rows_a,
                                              const int32_t* __restrict__ Zb, int nb, int rowb, int rows_b, int dk,
                                              int32_t* za, int ldza, int32_t* zb, int ldzb, F f) {
  for (int k0 = 0; k0 < dk; k0 += kCatTile) {
    const int kt = dk - k0 < kCatTile ? dk - k0 : kCatTile;
    __syncthreads();
    stage_cat_tile_T(Za, na, dk, k0, kt, rowa, rows_a, za, ldza);
    if (Zb) stage_cat_tile_T(Zb, nb, dk, k0, kt, rowb, rows_b, zb, ldzb);
    __syncthreads();
    f(k0, kt);
  }
}

// d2[i][j] += sum_{k < kt} w[k] [a_i[k] != b_j[k]] over one staged tile, w = the tile's inverse length scales.
template <typename Cfg, int TTM, int TTN>
__device__ __forceinline__ void tile_hamming(const int32_t* za, int ldza, const int32_t* zb, int ldzb,
                                             const double* __restrict__ w, int kt, int ty, int tx,
                                             double (&d2)[TTM][TTN]) {
  for (int k = 0; k < kt; ++k) {
    const double wk = __ldg(w + k);
#pragma unroll
    for (int i = 0; i < TTM; ++i) {
      const int av = za[k * ldza + Cfg::row_of(ty, i)];
#pragma unroll
      for (int j = 0; j < TTN; ++j) d2[i][j] += (av != zb[k * ldzb + Cfg::col_of(tx, j)]) ? wk : 0.0;
    }
  }
}

// lin[i][j] = sum_d (a_i[d] w_d - b)(b_j[d] w_d - b),  w_d = 1/length scale, b = coef*shift: the feature-scaled
// tfpk.Linear term of the `linear_coef` model (tuned_gp_models.py:220-230), a / b staged by stage_rows_T.
template <typename Cfg, int TTM, int TTN>
__device__ __forceinline__ void tile_lin(const double* sa, int lda, const double* sb, int ldb, const KernelParams& kp,
                                         int ty, int tx, double (&lin)[TTM][TTN]) {
#pragma unroll
  for (int i = 0; i < TTM; ++i)
#pragma unroll
    for (int j = 0; j < TTN; ++j) lin[i][j] = 0.0;
  for (int d = 0; d < kp.dc; ++d) {
    const double w = kp.inv_ls_c[d];
    double a[TTM], b[TTN];
#pragma unroll
    for (int i = 0; i < TTM; i += 2) {
      double2 t = *reinterpret_cast<const double2*>(sa + d * lda + Cfg::row_of(ty, i));
      a[i] = fma(t.x, w, -kp.lin_b); a[i + 1] = fma(t.y, w, -kp.lin_b);
    }
#pragma unroll
    for (int j = 0; j < TTN; j += 2) {
      double2 t = *reinterpret_cast<const double2*>(sb + d * ldb + Cfg::col_of(tx, j));
      b[j] = fma(t.x, w, -kp.lin_b); b[j + 1] = fma(t.y, w, -kp.lin_b);
    }
#pragma unroll
    for (int i = 0; i < TTM; ++i)
#pragma unroll
      for (int j = 0; j < TTN; ++j) lin[i][j] = fma(a[i], b[j], lin[i][j]);
  }
}

}  // namespace vzgp
