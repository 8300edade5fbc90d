// Dense fp64 linear algebra for the GP fit: Matern kernel matrices, blocked Cholesky with
// retry, triangular inverse by recursive doubling, K_y^-1, and the alpha solve.
//
// Replaces (reference, via TFP/XLA:CPU LAPACK): the covariance build and
// retrying_cholesky at vizier/_src/jax/models/tuned_gp_models.py:272-313 and the
// precompute in vizier/_src/jax/stochastic_process_model.py:968-997.
#include "launchers.h"
#include "tiles.cuh"

namespace vzgp {

using G64 = GemmCfg<64, 64, 16, 4, 4>;  // 256 threads, 4x4 register tile

// ---------------------------------------------------------------------------
// Kernel matrices
// ---------------------------------------------------------------------------
// K[i,j] = k(X_i, X_j) + diag_add*[i==j]; rows/cols >= n_valid -> identity.  One CTA per
// lower-triangular 64x64 tile; the mirrored tile is written too.
__global__ void __launch_bounds__(256) k_kernel_matrix(const double* __restrict__ X,
                                                       const int32_t* __restrict__ Z, int n,
                                                       int n_valid, KernelParams kp,
                                                       double diag_add, double* __restrict__ K,
                                                       int ldk) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  extern __shared__ double smem[];
  constexpr int LD = 66;
  double* sa = smem;
  double* sb = sa + kp.dc * LD;
  int32_t* za = reinterpret_cast<int32_t*>(sb + kp.dc * LD);
  int32_t* zb = za + kp.dk * LD;
  stage_rows_T(X, n, kp.dc, bi * 64, 64, sa, LD);
  stage_rows_T(X, n, kp.dc, bj * 64, 64, sb, LD);
  if (kp.dk > 0) {
    stage_rows_T_i32(Z, n, kp.dk, bi * 64, 64, za, LD);
    stage_rows_T_i32(Z, n, kp.dk, bj * 64, 64, zb, LD);
  }
  __syncthreads();
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
  double d2[4][4], unused[4][4];
  tile_d2<G64, 4, 4, false>(sa, LD, sb, LD, za, LD, zb, LD, kp, nullptr, ty, tx, d2, unused);
  if (kp.use_linear) tile_lin<G64, 4, 4>(sa, LD, sb, LD, kp, ty, tx, unused);   // `unused` now holds the linear term
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gi = bi * 64 + G64::row_of(ty, i), gj = bj * 64 + G64::col_of(tx, j);
      if (gi >= n || gj >= n) continue;
      double v;
      if (gi >= n_valid || gj >= n_valid) {
        v = (gi == gj) ? 1.0 : 0.0;
      } else {
        v = matern52(d2[i][j], kp.sf2);
        if (kp.use_linear) v = fma(kp.lin_a, unused[i][j], v);
        if (gi == gj) v += diag_add;
      }
      K[(size_t)gi * ldk + gj] = v;
      if (bi != bj) K[(size_t)gj * ldk + gi] = v;
    }
}

// Ks[m, j] = k(Xs_m, X_j) for m < M, j < n; columns j >= n_valid are written as 0.
using G128x64 = GemmCfg<128, 64, 16, 8, 4>;
__global__ void __launch_bounds__(256) k_cross_kernel(const double* __restrict__ Xs,
                                                      const int32_t* __restrict__ Zs, int M,
                                                      const double* __restrict__ X,
                                                      const int32_t* __restrict__ Z, int n,
                                                      int n_valid, KernelParams kp,
                                                      double* __restrict__ Ks, int ldks) {
  extern __shared__ double smem[];
  constexpr int LDA = 130, LDB = 66;
  double* sa = smem;
  double* sb = sa + kp.dc * LDA;
  int32_t* za = reinterpret_cast<int32_t*>(sb + kp.dc * LDB);
  int32_t* zb = za + kp.dk * LDA;
  const int m0 = blockIdx.y * 128, j0 = blockIdx.x * 64;
  stage_rows_T(Xs, M, kp.dc, m0, 128, sa, LDA);
  stage_rows_T(X, n, kp.dc, j0, 64, sb, LDB);
  if (kp.dk > 0) {
    stage_rows_T_i32(Zs, M, kp.dk, m0, 128, za, LDA);
    stage_rows_T_i32(Z, n, kp.dk, j0, 64, zb, LDB);
  }
  __syncthreads();
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
  double d2[8][4], unused[8][4];
  tile_d2<G128x64, 8, 4, false>(sa, LDA, sb, LDB, za, LDA, zb, LDB, kp, nullptr, ty, tx, d2,
                                unused);
  if (kp.use_linear) tile_lin<G128x64, 8, 4>(sa, LDA, sb, LDB, kp, ty, tx, unused);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gi = m0 + G128x64::row_of(ty, i), gj = j0 + G128x64::col_of(tx, j);
      if (gi >= M || gj >= n) continue;
      double v = matern52(d2[i][j], kp.sf2);
      if (kp.use_linear) v = fma(kp.lin_a, unused[i][j], v);
      Ks[(size_t)gi * ldks + gj] = gj < n_valid ? v : 0.0;
    }
}

// ---------------------------------------------------------------------------
// Cholesky: right-looking, 64-wide panels.
// ---------------------------------------------------------------------------
// L(lower) = A(lower) + shift*I, upper triangle zeroed; matrices are [np x ld], np % 64 == 0.
__global__ void k_copy_lower_shift(const double* __restrict__ A, int lda, int n_src, int np,
                                   double shift, double* __restrict__ L, int ldl) {
  int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= np) return;
  double v = 0.0;
  if (j <= i) {
    if (i < n_src && j < n_src) v = A[(size_t)i * lda + j];
    else v = (i == j) ? 1.0 : 0.0;
    if (i == j && i < n_src) v += shift;
  }
  L[(size_t)i * ldl + j] = v;
}

// Inverse of the lower-triangular 64x64 matrix a (shared memory, row stride 66) into x (same
// layout): column c is owned by 4 adjacent lanes (k-split), combined with two shuffles, so the 64
// dependent row steps need no block-wide barrier.  256 threads.
__device__ __forceinline__ void tri_inverse_64(const double* a, double* x, double* rdiag) {
  const int tid = threadIdx.x, c = tid >> 2, q = tid & 3;
  if (tid < 64) rdiag[tid] = 1.0 / a[tid * 66 + tid];
  __syncthreads();
  for (int i = 0; i < 64; ++i) {
    double s = 0.0;
    for (int k = c + q; k < i; k += 4) s = fma(a[i * 66 + k], x[k * 66 + c], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if (q == 0) x[i * 66 + c] = (c <= i) ? ((i == c ? 1.0 : 0.0) - s) * rdiag[i] : 0.0;
    __syncwarp();
  }
}

#ifdef VZ_POTF2_TIMING
__device__ long long g_potf2_t[32];
#define VZ_TSTAMP(i) do { if (threadIdx.x == 0) g_potf2_t[i] = clock64(); } while (0)
#endif
}  // namespace vzgp
#include "potf2.cuh"
namespace vzgp {

// Factor the 64x64 diagonal block kb in place (lower), zero its upper triangle, and write
// its inverse into the same block of Linv.  flag[0] is set to 1 if a pivot is not a
// positive finite number (the factor then holds NaN, like jnp.linalg.cholesky).  The work is
// potf2_inv_64 (potf2.cuh); 102 -> 18 us per block against the first column-by-column version.
__global__ void __launch_bounds__(256) k_potf2_inv(double* __restrict__ L, int ld, int kb,
                                                   double* __restrict__ Linv, int ldi,
                                                   int* __restrict__ flag) {
  extern __shared__ double smem[];
  constexpr int LD = 66;
  double* a = smem;              // [64][66]
  double* x = smem + 64 * LD;    // [64][66]
  double* t = x + 64 * LD;       // [32][34] temporary of the doubling steps
  __shared__ double rd[64];      // 1 / diagonal of the factor
  __shared__ int s_bad;
  double* blk = L + (size_t)kb * 64 * ld + kb * 64;
  const int tid = threadIdx.x;
  if (tid == 0) s_bad = 0;
  VZ_TSTAMP(0);
  {
    double2 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int e = tid + 256 * u, i = e >> 5, j2 = (e & 31) * 2;
      v[u] = *reinterpret_cast<const double2*>(blk + (size_t)i * ld + j2);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int e = tid + 256 * u, i = e >> 5, j2 = (e & 31) * 2;
      const bool upper_blk = (j2 >> 4) > (i >> 4);     // 16-blocks strictly above the diagonal
      *reinterpret_cast<double2*>(a + i * LD + j2) = upper_blk ? make_double2(0.0, 0.0) : v[u];
      *reinterpret_cast<double2*>(x + i * LD + j2) = make_double2(0.0, 0.0);
    }
  }
  __syncthreads();
  potf2_inv_64(a, x, t, rd, &s_bad);
  double* iblk = Linv + (size_t)kb * 64 * ldi + kb * 64;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int e = tid + 256 * u, i = e >> 5, j2 = (e & 31) * 2;
    *reinterpret_cast<double2*>(blk + (size_t)i * ld + j2) = *reinterpret_cast<const double2*>(a + i * LD + j2);
    *reinterpret_cast<double2*>(iblk + (size_t)i * ldi + j2) = *reinterpret_cast<const double2*>(x + i * LD + j2);
  }
  if (tid == 0 && s_bad) flag[0] = 1;
  VZ_TSTAMP(18);
}

// Panel solve as a GEMM with the inverted diagonal block:
//   L[i, kb] <- L[i, kb] * inv(L_kk)^T  for block rows i > kb  (in place; one CTA per block row).
__global__ void __launch_bounds__(256) k_trsm_panel(double* __restrict__ L, int ld, int kb,
                                                    const double* __restrict__ Linv, int ldi) {
  extern __shared__ double smem[];
  const int ib = kb + 1 + blockIdx.x;
  double acc[4][4] = {};
  const double* A = L + (size_t)kb * 64;                           // element (row, k) = L[row, kb*64+k]
  const double* B = Linv + (size_t)kb * 64 * ldi + (size_t)kb * 64; // element (j, k) = Linv_kk[j, k]
  gemm_mainloop<64, 64, 16, 4, 4, false, false>(A, ld, ib * 64, B, ldi, 0, 0, 64, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
  // every thread's reads of this block finished inside the main loop (it ends with a barrier)
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2) {
      double2 v = make_double2(acc[i][j], acc[i][j + 1]);
      *reinterpret_cast<double2*>(L + (size_t)(ib * 64 + G64::row_of(ty, i)) * ld + kb * 64 +
                                  G64::col_of(tx, j)) = v;
    }
}

// Trailing update  L[i, j] -= L[i, kb] * L[j, kb]^T  for kb < j <= i (lower tiles only), with
// look-ahead: the CTA that owns the NEXT
// diagonal block (kb+1, kb+1) keeps its updated tile in shared memory and factors + inverts it at once
// (potf2_inv_64), concurrently with the other tiles' updates.  The 64-pivot latency chain of the
// diagonal block thereby leaves the critical path of the blocked factorisation: per step
// trsm -> max(trailing update, diagonal factor) instead of factor -> trsm -> update.
__global__ void __launch_bounds__(256) k_syrk_potf2(double* __restrict__ L, int ld, int kb,
                                                    double* __restrict__ Linv, int ldi, int* __restrict__ flag) {
  extern __shared__ double smem[];
  const int ib = kb + 1 + blockIdx.y, jb = kb + 1 + blockIdx.x;
  if (jb > ib) return;
  double acc[4][4] = {};
  const double* P = L + (size_t)kb * 64;
  gemm_mainloop<64, 64, 16, 4, 4, false, false>(P, ld, ib * 64, P, ld, jb * 64, 0, 64, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
  if (blockIdx.x != 0 || blockIdx.y != 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; j += 2) {
        double2* p = reinterpret_cast<double2*>(L + (size_t)(ib * 64 + G64::row_of(ty, i)) * ld +
                                                jb * 64 + G64::col_of(tx, j));
        double2 v = *p;
        v.x -= acc[i][j];
        v.y -= acc[i][j + 1];
        *p = v;
      }
    return;
  }
  // ---- the next diagonal block: update in registers -> shared memory -> factor + invert ----
  constexpr int LD = 66;
  double* a = smem;              // [64][66]
  double* x = smem + 64 * LD;    // [64][66]
  double* t = x + 64 * LD;       // [32][34]
  __shared__ double rd[64];
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  double* blk = L + (size_t)ib * 64 * ld + ib * 64;
  __syncthreads();               // every warp is done with the GEMM staging buffers
  if (tid == 0) s_bad = 0;
  for (int e = tid; e < 64 * LD; e += 256) x[e] = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = G64::row_of(ty, i), c = G64::col_of(tx, j);
      const bool upper_blk = (c >> 4) > (r >> 4);
      a[r * LD + c] = upper_blk ? 0.0 : blk[(size_t)r * ld + c] - acc[i][j];
    }
  __syncthreads();
  potf2_inv_64(a, x, t, rd, &s_bad);
  double* iblk = Linv + (size_t)ib * 64 * ldi + ib * 64;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int e = tid + 256 * u, i = e >> 5, j2 = (e & 31) * 2;
    *reinterpret_cast<double2*>(blk + (size_t)i * ld + j2) = *reinterpret_cast<const double2*>(a + i * LD + j2);
    *reinterpret_cast<double2*>(iblk + (size_t)i * ldi + j2) = *reinterpret_cast<const double2*>(x + i * LD + j2);
  }
  if (tid == 0 && s_bad) flag[0] = 1;
}

// ---------------------------------------------------------------------------
// Triangular inverse by recursive doubling.  At level s (block size in elements,
// s = 64, 128, ...), for every aligned pair  [p, p+s) | [p+s, min(p+2s, np)):
//   X = -Binv * (C * Ainv),  C = L[right, left], Ainv/Binv = already inverted diagonal parts.
// Step 1 writes T = C*Ainv into the workspace, step 2 writes X into Linv[right, left].
// grid = (s/64 col tiles, s/64 row tiles, pairs); tiles outside the (possibly short) right
// part exit immediately.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_trtri_step1(const double* __restrict__ L, int ld,
                                                     const double* __restrict__ Linv, int ldi,
                                                     double* __restrict__ T, int ldt, int s,
                                                     int np) {
  extern __shared__ double smem[];
  const int p = blockIdx.z * 2 * s;
  const int r0 = p + s + blockIdx.y * 64;  // row tile in the right part
  const int c0 = p + blockIdx.x * 64;      // col tile in the left part
  if (r0 >= np || r0 >= p + 2 * s) return;
  double acc[4][4] = {};
  // T[i, j] = sum_{k>=j} C[i,k]*Ainv[k,j], k in [c0 - p, s) relative to p
  const double* A = L + (size_t)p;                       // (row, k) = L[row, p+k]
  const double* B = Linv + (size_t)p * ldi;              // (j, k)  = Linv[p+k, j]  (k-major)
  gemm_mainloop<64, 64, 16, 4, 4, false, true>(A, ld, r0, B, ldi, c0, c0 - p, s, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2)
      *reinterpret_cast<double2*>(T + (size_t)(r0 + G64::row_of(ty, i)) * ldt + c0 +
                                  G64::col_of(tx, j)) = make_double2(acc[i][j], acc[i][j + 1]);
}

__global__ void __launch_bounds__(256) k_trtri_step2(double* __restrict__ Linv, int ldi,
                                                     const double* __restrict__ T, int ldt, int s,
                                                     int np) {
  extern __shared__ double smem[];
  const int p = blockIdx.z * 2 * s;
  const int r0 = p + s + blockIdx.y * 64;
  const int c0 = p + blockIdx.x * 64;
  if (r0 >= np || r0 >= p + 2 * s) return;
  double acc[4][4] = {};
  // X[i, j] = -sum_{k<=i} Binv[i,k]*T[k,j], k relative to p+s in [0, r0-(p+s)+64)
  const double* A = Linv + (size_t)(p + s);              // (row, k) = Linv[row, p+s+k]
  const double* B = T + (size_t)(p + s) * ldt;           // (j, k)  = T[p+s+k, j]  (k-major)
  gemm_mainloop<64, 64, 16, 4, 4, false, true>(A, ldi, r0, B, ldt, c0, 0, r0 - (p + s) + 64, acc,
                                               smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2)
      *reinterpret_cast<double2*>(Linv + (size_t)(r0 + G64::row_of(ty, i)) * ldi + c0 +
                                  G64::col_of(tx, j)) = make_double2(-acc[i][j], -acc[i][j + 1]);
}

// Kinv = Linv^T Linv, lower tiles only:  Kinv[i,j] = sum_{k >= max(i,j)} Linv[k,i]*Linv[k,j].
// The tile (0,0) sums over all N rows - a 64-slab latency chain in one CTA - so the k range is cut
// into kLauumSplit planes: plane z holds the partial sum over k in [z*kc, (z+1)*kc) (only where that
// range meets k >= 64*ib); the consumer (k_nll_grad_tiles) adds the planes in ascending z.
__global__ void __launch_bounds__(256) k_lauum(const double* __restrict__ Linv, int ldi,
                                               double* __restrict__ Kinv, int ldk, int np, int kc) {
  extern __shared__ double smem[];
  const int ib = blockIdx.y, jb = blockIdx.x, z = blockIdx.z;
  if (jb > ib) return;
  const int k0 = max(ib * 64, z * kc), k1 = min(np, (z + 1) * kc);
  if (k0 >= k1) return;
  double acc[4][4] = {};
  gemm_mainloop<64, 64, 16, 4, 4, true, true>(Linv, ldi, ib * 64, Linv, ldi, jb * 64, k0, k1, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
  double* plane = Kinv + (size_t)z * np * ldk;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2) {
      const int gi = ib * 64 + G64::row_of(ty, i), gj = jb * 64 + G64::col_of(tx, j);
      *reinterpret_cast<double2*>(plane + (size_t)gi * ldk + gj) = make_double2(acc[i][j], acc[i][j + 1]);
    }
}

// ---------------------------------------------------------------------------
// Matrix-vector helpers (one warp per row), used for alpha = Linv^T (Linv y) and refinement.
// ---------------------------------------------------------------------------
// out[i] = sum_{j in [j_lo(i), j_hi(i))} M[i,j] * v[j];  mode 0: full row [0,ncols); 1: j <= i (lower
// triangular M); 2: j >= i (upper triangular M, e.g. L^-T from the dataflow factorisation).
__global__ void k_gemv_rows(const double* __restrict__ M, int ld, int nrows, int ncols,
                            const double* __restrict__ v, double* __restrict__ out, int lower_only) {
  int row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  int lane = threadIdx.x & 31;
  if (row >= nrows) return;
  int hi = lower_only == 1 ? row + 1 : ncols;
  int lo = lower_only == 2 ? (row & ~31) : 0;     // aligned start: the entries left of the diagonal are zero
  double s = 0.0;
  for (int j = lo + lane; j < hi; j += 32) s = fma(M[(size_t)row * ld + j], v[j], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (lane == 0) out[row] = s;
}

// out[j] = sum_{i >= j} M[i,j] * v[i]   (M lower triangular: out = M^T v).  One CTA per 64
// columns; 16 row groups of 64 threads stride the rows (coalesced 512-byte row segments), then a
// fixed-order shared-memory reduction.
__global__ void __launch_bounds__(1024) k_gemv_lower_T(const double* __restrict__ M, int ld, int np,
                                                       const double* __restrict__ v,
                                                       double* __restrict__ out) {
  __shared__ double part[16][64];
  const int c = threadIdx.x & 63, g = threadIdx.x >> 6;
  const int j = blockIdx.x * 64 + c;
  double s = 0.0;
  for (int i = blockIdx.x * 64 + g; i < np; i += 16)
    if (i >= j) s = fma(M[(size_t)i * ld + j], v[i], s);
  part[g][c] = s;
  __syncthreads();
  if (g == 0) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 16; ++k) t += part[k][c];
    out[j] = t;
  }
}

// r = y - Ky * a  (Ky symmetric, full storage)
__global__ void k_residual(const double* __restrict__ Ky, int ld, int np, const double* __restrict__ y,
                           const double* __restrict__ a, double* __restrict__ r) {
  int row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  int lane = threadIdx.x & 31;
  if (row >= np) return;
  double s = 0.0;
  for (int j = lane; j < np; j += 32) s = fma(Ky[(size_t)row * ld + j], a[j], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (lane == 0) r[row] = y[row] - s;
}

__global__ void k_axpy(int n, double a, const double* __restrict__ x, double* __restrict__ y) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = fma(a, x[i], y[i]);
}

__global__ void k_pad_vector(const double* __restrict__ src, int n, int n_valid, int np,
                             double* __restrict__ dst, double offset) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < np) dst[i] = (i < n && i < n_valid) ? src[i] - offset : 0.0;   // offset: constant prior mean
}

__global__ void k_pad_rows(const double* __restrict__ src, int n, int d, int np,
                           double* __restrict__ dst) {
  size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)np * d) return;
  dst[e] = e < (size_t)n * d ? src[e] : 0.0;
}

// XT[0][d][i] = X[i][d] * inv_ls[d],  XT[1][d][i] = X[i][d]   (X is [np x dc], already padded)
__global__ void k_transpose_scale(const double* __restrict__ X, int np, int dc, KernelParams kp,
                                  double* __restrict__ XT) {
  size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)np * dc) return;
  int d = (int)(e / np), i = (int)(e % np);
  double v = X[(size_t)i * dc + d];
  XT[e] = v * kp.inv_ls_c[d];
  XT[(size_t)np * dc + e] = v;
}

__global__ void k_pad_rows_i32(const int32_t* __restrict__ src, int n, int d, int np,
                               int32_t* __restrict__ dst) {
  size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)np * d) return;
  dst[e] = e < (size_t)n * d ? src[e] : -1;
}

// n_metrics * sum_i log L_ii over i < n and  0.5 * sum_m sum_i w_m[i]^2 over i < n_valid  ->  out[0], out[1]
// (single block; w_m = w + m * wstride: the independent multi-task GP shares one factor).
// out[2] = sum_i alpha[i] over the valid rows (gradient of the constant mean of the linear_coef model).
// The log-det runs over all n observations, masked ones included: a masked row is an identity row, so it adds
// log(1 + shift) once the jitter fires, as in TFP's masked GaussianProcess (DESIGN.md, deviations).
__global__ void k_logdet_quad(const double* __restrict__ L, int ld, int n, int n_valid,
                              const double* __restrict__ w, int wstride, int n_metrics, double* __restrict__ out,
                              const double* __restrict__ alpha) {
  __shared__ double red[32];
  double a = 0.0, b = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    a += log(L[(size_t)i * ld + i]);
    if (i >= n_valid) continue;
    for (int m = 0; m < n_metrics; ++m) { const double v = w[(size_t)m * wstride + i]; b = fma(v, v, b); }
    if (alpha) c += alpha[i];
  }
  a = block_sum(a, red);
  b = block_sum(b, red);
  c = block_sum(c, red);
  if (threadIdx.x == 0) { out[0] = n_metrics * a; out[1] = 0.5 * b; out[2] = c; }
}

// ---------------------------------------------------------------------------
// Host drivers
// ---------------------------------------------------------------------------
static size_t kernel_smem_bytes(int dc, int dk, int rows_a, int rows_b) {
  return sizeof(double) * dc * (rows_a + 2 + rows_b + 2) + sizeof(int32_t) * dk * (rows_a + 2 + rows_b + 2);
}

int fill_kernel_params(const vzgp_params* p, int dc, int dk, KernelParams* kp) {
  VZ_ARG(p != nullptr, "params");
  VZ_ARG(dc >= 0 && dc <= kMaxDc, "Dc out of range [0,64]");
  VZ_ARG(dk >= 0 && dk <= kMaxDk, "Dk out of range [0,32]");
  VZ_ARG(dc + dk > 0, "no features");
  VZ_ARG(dc == 0 || p->continuous_length_scale_squared != nullptr, "continuous length scales");
  VZ_ARG(dk == 0 || p->categorical_length_scale_squared != nullptr, "categorical length scales");
  kp->dc = dc;
  kp->dk = dk;
  kp->sf2 = p->signal_variance;
  for (int d = 0; d < kMaxDc; ++d) {
    kp->inv_ls2_c[d] = d < dc ? 1.0 / p->continuous_length_scale_squared[d] : 0.0;
    kp->inv_ls_c[d] = d < dc ? 1.0 / std::sqrt(p->continuous_length_scale_squared[d]) : 0.0;
  }
  for (int d = 0; d < kMaxDk; ++d)
    kp->inv_ls2_k[d] = d < dk ? 1.0 / p->categorical_length_scale_squared[d] : 0.0;
  kp->use_linear = p->linear_coef != 0.0 ? 1 : 0;
  kp->lin_a = kp->use_linear ? (p->linear_coef * p->linear_slope_amplitude) * (p->linear_coef * p->linear_slope_amplitude) : 0.0;
  kp->lin_b = kp->use_linear ? p->linear_coef * p->linear_shift : 0.0;
  return 0;
}

// The captured NLL graph re-parameterises these kernels by argument position (c_abi.cu): pin the positions.
static_assert(KernelArgs<decltype(&k_kernel_matrix)>::count == kKernelMatrixArgs &&
              std::is_same<KernelArgs<decltype(&k_kernel_matrix)>::arg<kKernelMatrixKpArg>, KernelParams>::value &&
              std::is_same<KernelArgs<decltype(&k_kernel_matrix)>::arg<kKernelMatrixDiagArg>, double>::value,
              "k_kernel_matrix signature changed: update kKernelMatrix*Arg in launchers.h");
static_assert(KernelArgs<decltype(&k_transpose_scale)>::count == kTransposeScaleArgs &&
              std::is_same<KernelArgs<decltype(&k_transpose_scale)>::arg<kTransposeScaleKpArg>, KernelParams>::value,
              "k_transpose_scale signature changed: update kTransposeScale*Arg in launchers.h");
const void* kernel_matrix_func() { return reinterpret_cast<const void*>(&k_kernel_matrix); }
const void* transpose_scale_func() { return reinterpret_cast<const void*>(&k_transpose_scale); }

int launch_kernel_matrix(vzgp_handle* h, const double* X, const int32_t* Z, int n, int n_valid,
                         const KernelParams& kp, double diag_add, double* K, int ldk) {
  int nb = (n + 63) / 64;
  size_t sm = kernel_smem_bytes(kp.dc, kp.dk, 64, 64);
  VZ_TRY(raise_dyn_smem((const void*)k_kernel_matrix, sm));
  k_kernel_matrix<<<dim3(nb, nb), 256, sm, h->stream>>>(X, Z, n, n_valid, kp, diag_add, K, ldk);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int launch_cross_kernel(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const double* X,
                        const int32_t* Z, int n, int n_valid, const KernelParams& kp, double* Ks,
                        int ldks) {
  size_t sm = kernel_smem_bytes(kp.dc, kp.dk, 128, 64);
  VZ_TRY(raise_dyn_smem((const void*)k_cross_kernel, sm));
  dim3 grid((n + 63) / 64, (M + 127) / 128);
  k_cross_kernel<<<grid, 256, sm, h->stream>>>(Xs, Zs, M, X, Z, n, n_valid, kp, Ks, ldks);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// Factor `L` in place (already holds the shifted lower triangle, np % 64 == 0) and fill the
// diagonal blocks of Linv.  flag (device int) is raised on a bad pivot.
constexpr size_t kDiagSmem = sizeof(double) * (2 * 64 * 66 + 32 * 34);

int potrf_blocked(vzgp_handle* h, double* L, int ld, double* Linv, int ldi, int np, int* flag) {
  const int nb = np / 64;
  VZ_CUDA(cudaFuncSetAttribute(k_potf2_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDiagSmem));
  const size_t sm = G64::kSmemBytes;
  const size_t sm2 = sm > kDiagSmem ? sm : kDiagSmem;
  VZ_TRY(raise_dyn_smem((const void*)k_syrk_potf2, sm2));
  // Right-looking with one block of look-ahead: block 0 is factored alone; afterwards the trailing
  // update of step kb also factors diagonal block kb+1 (k_syrk_potf2).
  k_potf2_inv<<<1, 256, kDiagSmem, h->stream>>>(L, ld, 0, Linv, ldi, flag);
  VZ_CHECK_LAUNCH();
  h->launches++;
  for (int kb = 0; kb + 1 < nb; ++kb) {
    const int rem = nb - kb - 1;
    k_trsm_panel<<<rem, 256, sm, h->stream>>>(L, ld, kb, Linv, ldi);
    VZ_CHECK_LAUNCH();
    k_syrk_potf2<<<dim3(rem, rem), 256, sm2, h->stream>>>(L, ld, kb, Linv, ldi, flag);
    VZ_CHECK_LAUNCH();
    h->launches += 2;
  }
  return 0;
}

// Complete Linv (diagonal 64-blocks already inverted by potrf_blocked or k_potf2_inv).
int trtri_doubling(vzgp_handle* h, const double* L, int ld, double* Linv, int ldi, double* T,
                   int ldt, int np) {
  const size_t sm = G64::kSmemBytes;
  for (int s = 64; s < np; s *= 2) {
    int pairs = (np + 2 * s - 1) / (2 * s);
    dim3 grid(s / 64, s / 64, pairs);
    k_trtri_step1<<<grid, 256, sm, h->stream>>>(L, ld, Linv, ldi, T, ldt, s, np);
    VZ_CHECK_LAUNCH();
    k_trtri_step2<<<grid, 256, sm, h->stream>>>(Linv, ldi, T, ldt, s, np);
    VZ_CHECK_LAUNCH();
    h->launches += 2;
  }
  return 0;
}

int lauum_plane_rows(int np) { return ((np / 64 + kLauumSplit - 1) / kLauumSplit) * 64; }

int launch_lauum(vzgp_handle* h, const double* Linv, int ldi, double* Kinv, int ldk, int np) {
  const int nb = np / 64;
  k_lauum<<<dim3(nb, nb, kLauumSplit), 256, G64::kSmemBytes, h->stream>>>(Linv, ldi, Kinv, ldk, np, lauum_plane_rows(np));
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// plane 0 (lower tiles) += planes 1..kLauumSplit-1 that meet the tile's k range (see k_lauum)
__global__ void k_sum_planes(double* __restrict__ Kinv, int np, int kc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j > i || j >= np) return;
  const int bi = i / 64;
  double s = 0.0;
  for (int z = (bi * 64) / kc; z < kLauumSplit && z * kc < np; ++z) s += Kinv[((size_t)z * np + i) * np + j];
  Kinv[(size_t)i * np + j] = s;
}
int launch_sum_planes(vzgp_handle* h, double* Kinv, int np, int kc) {
  k_sum_planes<<<dim3((np + 255) / 256, np), 256, 0, h->stream>>>(Kinv, np, kc);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int launch_copy_lower_shift(vzgp_handle* h, const double* A, int lda, int n_src, int np,
                            double shift, double* L, int ldl) {
  k_copy_lower_shift<<<dim3((np + 255) / 256, np), 256, 0, h->stream>>>(A, lda, n_src, np, shift, L, ldl);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// Inverts the diagonal 64-blocks of an already-triangular L (for vzgp_tri_inverse): reuse
// k_potf2_inv's substitution by a dedicated light kernel.
__global__ void __launch_bounds__(256) k_diag_inv(const double* __restrict__ L, int ld,
                                                  double* __restrict__ Linv, int ldi) {
  extern __shared__ double smem[];
  double* a = smem;
  double* x = smem + 64 * 66;
  const int kb = blockIdx.x, tid = threadIdx.x;
  const double* blk = L + (size_t)kb * 64 * ld + kb * 64;
  for (int e = tid; e < 64 * 64; e += 256) a[(e >> 6) * 66 + (e & 63)] = blk[(size_t)(e >> 6) * ld + (e & 63)];
  __syncthreads();
  __shared__ double rdiag[64];
  tri_inverse_64(a, x, rdiag);
  __syncthreads();
  double* iblk = Linv + (size_t)kb * 64 * ldi + kb * 64;
  for (int e = tid; e < 64 * 64; e += 256) {
    int i = e >> 6, j = e & 63;
    iblk[(size_t)i * ldi + j] = (j <= i) ? x[i * 66 + j] : 0.0;
  }
}

int launch_diag_inv(vzgp_handle* h, const double* L, int ld, double* Linv, int ldi, int np) {
  VZ_CUDA(cudaFuncSetAttribute(k_diag_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDiagSmem));
  k_diag_inv<<<np / 64, 256, kDiagSmem, h->stream>>>(L, ld, Linv, ldi);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int launch_gemv_rows(vzgp_handle* h, const double* M, int ld, int np, const double* v, double* out,
                     int lower_only, int ncols) {
  k_gemv_rows<<<(np + 7) / 8, 256, 0, h->stream>>>(M, ld, np, ncols > 0 ? ncols : np, v, out, lower_only);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_gemv_lower_T(vzgp_handle* h, const double* M, int ld, int np, const double* v, double* out) {
  k_gemv_lower_T<<<np / 64, 1024, 0, h->stream>>>(M, ld, np, v, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_residual(vzgp_handle* h, const double* Ky, int ld, int np, const double* y, const double* a,
                    double* r) {
  k_residual<<<(np + 7) / 8, 256, 0, h->stream>>>(Ky, ld, np, y, a, r);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_axpy(vzgp_handle* h, int n, double a, const double* x, double* y) {
  k_axpy<<<(n + 255) / 256, 256, 0, h->stream>>>(n, a, x, y);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
__global__ void k_add_scalar(int n, double a, double* __restrict__ y) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] += a;
}
int launch_add_scalar(vzgp_handle* h, int n, double a, double* y) {
  k_add_scalar<<<(n + 255) / 256, 256, 0, h->stream>>>(n, a, y);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_pad_vector(vzgp_handle* h, const double* src, int n, int n_valid, int np, double* dst, double offset) {
  k_pad_vector<<<(np + 255) / 256, 256, 0, h->stream>>>(src, n, n_valid, np, dst, offset);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_pad_rows(vzgp_handle* h, const double* src, int n, int d, int np, double* dst) {
  size_t tot = (size_t)np * d;
  if (tot == 0) return 0;
  k_pad_rows<<<(unsigned)((tot + 255) / 256), 256, 0, h->stream>>>(src, n, d, np, dst);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_transpose_scale(vzgp_handle* h, const double* X, int np, int dc, const KernelParams& kp,
                           double* XT) {
  size_t tot = (size_t)np * dc;
  if (tot == 0) return 0;
  k_transpose_scale<<<(unsigned)((tot + 255) / 256), 256, 0, h->stream>>>(X, np, dc, kp, XT);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_pad_rows_i32(vzgp_handle* h, const int32_t* src, int n, int d, int np, int32_t* dst) {
  size_t tot = (size_t)np * d;
  if (tot == 0) return 0;
  k_pad_rows_i32<<<(unsigned)((tot + 255) / 256), 256, 0, h->stream>>>(src, n, d, np, dst);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_logdet_quad(vzgp_handle* h, const double* L, int ld, int n, int n_valid, const double* w,
                       double* out, int wstride, int n_metrics, const double* alpha) {
  k_logdet_quad<<<1, 256, 0, h->stream>>>(L, ld, n, n_valid, w, wstride, n_metrics, out, alpha);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}


// ---------------------------------------------------------------------------
// Joint posterior over a few query points (predict/sample path, not the hot loop):
//   W = K* Linv^T  (triangular: k <= j),   cov = K** - W W^T.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gemm_nt_tri(const double* __restrict__ A, int lda,
                                                     const double* __restrict__ B, int ldb,
                                                     double* __restrict__ C, int ldc) {
  extern __shared__ double smem[];
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  double acc[4][4] = {};
  gemm_mainloop<64, 64, 16, 4, 4, false, false>(A, lda, i0, B, ldb, j0, 0, j0 + 64, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2)
      *reinterpret_cast<double2*>(C + (size_t)(i0 + G64::row_of(ty, i)) * ldc + j0 + G64::col_of(tx, j)) =
          make_double2(acc[i][j], acc[i][j + 1]);
}

// C[i,j] = C[i,j] - sum_k W[i,k] W[j,k] + diag_add*[i==j]
__global__ void __launch_bounds__(256) k_cov_update(const double* __restrict__ W, int ldw, int kdim,
                                                    double* __restrict__ C, int ldc, double diag_add) {
  extern __shared__ double smem[];
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  double acc[4][4] = {};
  gemm_mainloop<64, 64, 16, 4, 4, false, false>(W, ldw, i0, W, ldw, j0, 0, kdim, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gi = i0 + G64::row_of(ty, i), gj = j0 + G64::col_of(tx, j);
      double* p = C + (size_t)gi * ldc + gj;
      *p = *p - acc[i][j] + (gi == gj ? diag_add : 0.0);
    }
}

int launch_gemm_nt_tri(vzgp_handle* h, const double* A, int lda, int mp, const double* B, int ldb,
                       int np, double* C, int ldc) {
  k_gemm_nt_tri<<<dim3(np / 64, mp / 64), 256, G64::kSmemBytes, h->stream>>>(A, lda, B, ldb, C, ldc);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}
int launch_cov_update(vzgp_handle* h, const double* W, int ldw, int kdim, int mp, double* C, int ldc,
                      double diag_add) {
  k_cov_update<<<dim3(mp / 64, mp / 64), 256, G64::kSmemBytes, h->stream>>>(W, ldw, kdim, C, ldc, diag_add);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
