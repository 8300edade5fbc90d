// Pieces of the scoring path shared by score.cu (stand-alone kernels) and eagle_grid.cu (the
// multi-CTA persistent acquisition-optimiser loop): the argument block, the final-score formula and the
// trial-axis kernels for small candidate pools as device functions.
#pragma once
#include <cuda.h>

#include "acq_fn.cuh"
#include "async.cuh"
#include "launchers.h"
#include "tiles.cuh"

namespace vzgp {

constexpr int kTM = 64;          // candidates per tile
constexpr int kLD1 = 66;         // phase-1 smem row stride (64 rows/cols + 2)

struct ScoreArgs {
  // TMA descriptors (must stay first: 64-byte alignment inside the __grid_constant__ parameter).
  alignas(64) CUtensorMap mapA;  // scratch  as [gridDim.x*64 rows][np], box 64 x 16, SWIZZLE_128B
  alignas(64) CUtensorMap mapB;  // Linv     as [np rows][np],           box 128 x 16, SWIZZLE_128B
  const double* Xs;
  const int32_t* Zs;
  int M;
  const double* XT;   // [2][dc][np]: scaled / unscaled transposed trials
  const int32_t* Z;
  int np;
  int n_valid;
  const double* Linv;
  int ldi;
  const double* alpha;
  KernelParams kp;
  double sn2;
  TrustRegion tr;
  double* scratch;  // [gridDim.x][64][np]
  int nsplit;       // > 1: output column blocks of one tile are shared by nsplit CTAs (small M)
  double* part;     // nsplit > 1: [nsplit + 2][Mpad] partial row sums, then mu, then linf
  int mpad;
  // small-pool path (k_cross_small / k_var_small / k_small_finalize)
  double* part_rs;    // [np/16][Mpad] partial row sums of W^2, one row per 16-column block
  double* part_mu;    // [np/64][Mpad] partial means, one row per 64-trial block
  double* part_linf;  // [np/64][Mpad] partial trust-region distances
  int box_rows;       // rows of the K* TMA box (small-pool W phase)
  int use_tma;        // small-pool W phase: TMA boxes instead of cp.async
  double* score;
  double* mu;
  double* sigma;
  double* linf;
  int* clamp_count;
  AcqFn acq;          // acquisition function of (mean, stddev)
};

// Final score from the reduced pieces (shared by the fused epilogue and the split finalize kernel).
template <bool GENERIC = true>
__device__ __forceinline__ void emit_score(const ScoreArgs& a, int m, double rs, double mean, double dist,
                                           int& clamped) {
  double var = a.kp.sf2 - rs + a.sn2;
  if (var < 0.0) { var = 0.0; ++clamped; }
  const double sd = sqrt(var);
  a.score[m] = tr_apply(a.tr, acq_eval<GENERIC>(a.acq, mean, sd), dist);
  if (a.mu) a.mu[m] = mean;
  if (a.sigma) a.sigma[m] = sd;
  if (a.linf) a.linf[m] = dist;
}

// ---------------------------------------------------------------------------
// Small candidate pools (the acquisition optimiser scores 25..1000 candidates per iteration,
// vectorized_base.py:431-495).  One persistent CTA per 64-candidate tile leaves the GPU empty there,
// so the work is cut along the TRIAL axis instead:
//   k_cross_small  grid (np/64, tiles): K* block [64 cand x 64 trials] -> scratch, partial mean / L-inf
//   k_var_small    grid (np/16, tiles): W[:, 16 cols] = K*[:, 0:kext] Linv[16 rows, 0:kext]^T on the
//                  DMMA pipe (cp.async ring), partial row sums of W^2
//   k_small_finalize: fixed-order sums of the partials -> variance, acquisition, trust region.
// All reductions have a fixed order: results are reproducible run to run.
// ---------------------------------------------------------------------------
constexpr int kSmallThreads = 256;
constexpr int kVarCols = 8;            // output columns per k_var_small work item (one DMMA n-tile)
constexpr int kVarBK = 64;             // k-slab
constexpr int kVarLD = 72;             // smem row stride (doubles, = 8 mod 16): 16-byte fragment loads are conflict-free
constexpr int kVarStages = 4;
constexpr int kVarStageDoubles = (kTM + kVarCols) * kVarLD;

// K* block (candidates of `tile` x 64 trials of block jb), partial mean / L-inf.  256 threads; only the
// first NI groups of 16 candidate rows hold real candidates (a 25-candidate batch computes 32 rows).
template <bool WITH_LINF, int NI>
__device__ __forceinline__ void cross_small_core(const ScoreArgs& a, int jb, int tile, int rg, double* smem_raw) {
  constexpr int LD = kLD1;
  const int dc = a.kp.dc, dk = a.kp.dk, np = a.np;
  double* sa = smem_raw;                 // [dc][LD] candidates (transposed)
  double* sb = sa + dc * LD;             // [dc][LD] trials
  int32_t* za = reinterpret_cast<int32_t*>(sb + dc * LD);   // [dk][LD]
  int32_t* zb = za + dk * LD;
  const int tid = threadIdx.x;
  const int m0 = tile * kTM;
  const int ty = (tid >> 4) + 16 * rg, tx = tid & 15;       // rows ty + 16 i, columns 4 tx + j
  for (int e = tid; e < kTM * dc; e += kSmallThreads) {
    const int r = e / dc, d = e - r * dc;
    const int gr = m0 + r;
    const double v = gr < a.M ? __ldg(a.Xs + (size_t)gr * dc + d) : 0.0;
    sa[d * LD + r] = WITH_LINF ? v : v * a.kp.inv_ls_c[d];
  }
  {
    const double* src = (WITH_LINF ? a.XT + (size_t)dc * np : a.XT) + jb * 64;
    for (int e = tid; e < dc * 32; e += kSmallThreads) {
      const int d = e >> 5, q = e & 31;
      *reinterpret_cast<double2*>(sb + d * LD + 2 * q) = __ldg(reinterpret_cast<const double2*>(src + (size_t)d * np + 2 * q));
    }
  }
  if (dk > 0) {
    stage_rows_T_i32(a.Zs, a.M, dk, m0, kTM, za, LD, kSmallThreads);
    stage_rows_T_i32(a.Z, np, dk, jb * 64, 64, zb, LD, kSmallThreads);
  }
  __syncthreads();
  double d2[NI][4], lf[NI][4];
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { d2[i][j] = 0.0; lf[i][j] = 0.0; }
  for (int d = 0; d < dc; ++d) {
    double aa[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) aa[i] = sa[d * LD + ty + 16 * i];
    const double2 b0 = *reinterpret_cast<const double2*>(sb + d * LD + 4 * tx);
    const double2 b1 = *reinterpret_cast<const double2*>(sb + d * LD + 4 * tx + 2);
    const double bb[4] = {b0.x, b0.y, b1.x, b1.y};
    if (WITH_LINF) {
      const double w = a.kp.inv_ls2_c[d];
      const bool in_tr = a.tr.mask[d] != 0;
#pragma unroll
      for (int i = 0; i < NI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double df = aa[i] - bb[j];
          d2[i][j] = fma(df * df, w, d2[i][j]);
          if (in_tr) lf[i][j] = fmax(lf[i][j], fabs(df));
        }
    } else {
#pragma unroll
      for (int i = 0; i < NI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double df = aa[i] - bb[j];
          d2[i][j] = fma(df, df, d2[i][j]);
        }
    }
  }
  for (int k = 0; k < dk; ++k) {
    const double w = a.kp.inv_ls2_k[k];
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int avz = za[k * LD + ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) d2[i][j] += (avz != zb[k * LD + 4 * tx + j]) ? w : 0.0;
    }
  }
  double* scr = a.scratch + (size_t)tile * kTM * np + jb * 64;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int r = ty + 16 * i;
    double kv[4], mu_part = 0.0, lmin = INFINITY;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gc = jb * 64 + 4 * tx + j;
      kv[j] = gc < a.n_valid ? matern52(d2[i][j], a.kp.sf2) : 0.0;
      mu_part = fma(kv[j], __ldg(a.alpha + gc), mu_part);
      if (WITH_LINF && gc < a.tr.rows) lmin = fmin(lmin, lf[i][j]);
    }
    *reinterpret_cast<double2*>(scr + (size_t)r * np + 4 * tx) = make_double2(kv[0], kv[1]);
    *reinterpret_cast<double2*>(scr + (size_t)r * np + 4 * tx + 2) = make_double2(kv[2], kv[3]);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      mu_part += __shfl_xor_sync(0xffffffffu, mu_part, o);
      if (WITH_LINF) lmin = fmin(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
    }
    if (tx == 0) {
      a.part_mu[(size_t)jb * a.mpad + m0 + r] = mu_part;
      a.part_linf[(size_t)jb * a.mpad + m0 + r] = lmin;
    }
  }
}

// Work item (jb, tile, rg): 16 candidates (row group rg of the tile) x 64 trials.  Items whose row group
// holds no real candidate return at once.
template <bool WITH_LINF>
__device__ __forceinline__ void cross_small_block(const ScoreArgs& a, int jb, int tile, int rg, double* smem_raw) {
  const int rows = min(kTM, a.M - tile * kTM);
  if (rg * 16 >= rows) return;
  cross_small_core<WITH_LINF, 1>(a, jb, tile, rg, smem_raw);
}

#ifdef VZ_EAGLE_TIMING
__device__ long long g_var_t[8];
#define VZ_VT(i) do { if (threadIdx.x == 0 && b == a.np / kVarCols - 1) { long long t1_ = clock64(); atomicAdd((unsigned long long*)&g_var_t[i], (unsigned long long)(t1_ - t0_)); t0_ = t1_; } } while (0)
#else
#define VZ_VT(i) do {} while (0)
#endif
// W[:, 8 columns of block b] for `tile`, partial row sums of W^2.  256 threads.
// The work is bound by what ONE SM can pull from L2 (the last block reads (rows + 8) x N doubles) and by
// the issue rate of a single DMMA warp per scheduler, so: narrow column blocks (more CTAs, less data
// each), and when the tile has <= 32 candidates warps 4..7 do nothing but issue the cp.async copies
// while warps 0..3 run the DMMAs - the two no longer serialise inside one instruction stream.
__device__ __forceinline__ void var_small_block(const ScoreArgs& a, int b, int tile, double* smem_raw) {
  const int np = a.np;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int m0 = tile * kTM;
  const int rows = min(kTM, a.M - m0);
#ifdef VZ_EAGLE_TIMING
  long long t0_ = clock64();
#endif
  const int nmt = (rows + 7) >> 3;                 // m-tiles (8 candidates) that hold real rows
  const int kext = kVarCols * (b + 1);             // Linv[j, k] = 0 for k > j
  const int nslab = (kext + kVarBK - 1) / kVarBK;
  const double* Asrc = a.scratch + (size_t)tile * kTM * np;
  const double* Bsrc = a.Linv + (size_t)b * kVarCols * a.ldi;
  // One slab = (nmt*8 rows of K*) + (8 rows of Linv), 64 doubles = 32 16-byte chunks per row.  A copying
  // thread always takes chunk column (t & 31) of rows (t >> 5) + nw*u: one add per slab of address work.
  const int nrows = nmt * 8 + kVarCols;
  const bool split = nmt <= 4;                     // warps 4..7 copy, warps 0..3 compute
  const bool copier = !split || warp >= 4;
  const int cq = tid & 31, nw = split ? 4 : 8, r0 = split ? warp - 4 : warp;
  auto issue = [&](int ks) {
    double* stg = smem_raw + (ks % kVarStages) * kVarStageDoubles;
    const int koff = ks * kVarBK + 2 * cq;
    for (int rr = r0; rr < nrows; rr += nw) {
      const bool is_a = rr < nmt * 8;
      const double* src = is_a ? Asrc + (size_t)rr * np : Bsrc + (size_t)(rr - nmt * 8) * a.ldi;
      const int drow = is_a ? rr : kTM + rr - nmt * 8;
      cp_async16(stg + drow * kVarLD + 2 * cq, src + koff, true);
    }
  };
#pragma unroll
  for (int s = 0; s < kVarStages - 1; ++s) {
    if (copier && s < nslab) issue(s);
    cp_async_commit();
  }
  double acc[4][2];   // four independent k chains
#pragma unroll
  for (int q = 0; q < 4; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
  VZ_VT(0);
  for (int ks = 0; ks < nslab; ++ks) {
    cp_async_wait<kVarStages - 2>();
    VZ_VT(1);
    __syncthreads();                         // slab ks landed for everyone; slab ks-1 fully consumed
    VZ_VT(2);
    if (copier && ks + kVarStages - 1 < nslab) issue(ks + kVarStages - 1);
    cp_async_commit();
    VZ_VT(3);
    if (warp < nmt) {
      const double* stg = smem_raw + (ks % kVarStages) * kVarStageDoubles;
      const double* Ar = stg + (warp * 8 + fr) * kVarLD + 2 * fk;
      const double* Br = stg + (kTM + fr) * kVarLD + 2 * fk;
#pragma unroll
      for (int h = 0; h < kVarBK / 8; ++h) {
        const double2 av = *reinterpret_cast<const double2*>(Ar + 8 * h);
        const double2 bv = *reinterpret_cast<const double2*>(Br + 8 * h);
        const int c = (h & 1) * 2;
        dmma_8x8x4(acc[c][0], acc[c][1], av.x, bv.x);
        dmma_8x8x4(acc[c + 1][0], acc[c + 1][1], av.y, bv.y);
      }
    }
    VZ_VT(4);
  }
  cp_async_wait<0>();
  if (warp < nmt) {
    double rs = 0.0;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const double w = (acc[0][e] + acc[1][e]) + (acc[2][e] + acc[3][e]);
      rs = fma(w, w, rs);
    }
    rs += __shfl_xor_sync(0xffffffffu, rs, 1);
    rs += __shfl_xor_sync(0xffffffffu, rs, 2);
    if (fk == 0) a.part_rs[(size_t)b * a.mpad + m0 + warp * 8 + fr] = rs;
  }
}

// The same work item with the operands fetched by the TMA unit: per 64-wide slab four K* boxes
// (box_rows x 16 doubles) and four Linv boxes (8 x 16 doubles), 128-byte swizzle, one elected thread
// issues them and a per-stage mbarrier counts the bytes; the DMMA warps read the swizzled fragments as in
// k_score.  No per-thread copy instructions at all.
constexpr int kVarTmaStageDoubles = (kTM + kVarCols) * kVarBK;    // dense boxes
__device__ __forceinline__ void var_small_block_tma(const ScoreArgs& a, int b, int tile, double* smem_raw) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;
  const int m0 = tile * kTM;
  const int rows = min(kTM, a.M - m0);
  const int nmt = (rows + 7) >> 3;
  const int kext = kVarCols * (b + 1);
  const int nslab = (kext + kVarBK - 1) / kVarBK;
  double* base = smem_raw + (((1024u - (static_cast<unsigned>(__cvta_generic_to_shared(smem_raw)) & 1023u)) & 1023u) >> 3);
  const int abox = a.box_rows * 16;                 // doubles per K* box
  __shared__ uint64_t full_bar[kVarStages];
  if (tid == 0) {
    for (int s2 = 0; s2 < kVarStages; ++s2) mbar_init(full_bar + s2, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  fence_proxy_async();            // K* was written through the generic proxy (previous phase / kernel)
  __syncthreads();
  auto issue = [&](int ks) {      // one thread
    const int stage = ks % kVarStages;
    double* stg = base + stage * kVarTmaStageDoubles;
    mbar_expect_tx(full_bar + stage, (unsigned)((a.box_rows + kVarCols) * kVarBK * sizeof(double)));
#pragma unroll
    for (int q = 0; q < kVarBK / 16; ++q) {
      tma_load_2d(stg + q * abox, &a.mapA, ks * kVarBK + 16 * q, tile * kTM, full_bar + stage);
      tma_load_2d(stg + 4 * abox + q * kVarCols * 16, &a.mapB, ks * kVarBK + 16 * q, b * kVarCols, full_bar + stage);
    }
  };
  if (tid == 0)
    for (int s2 = 0; s2 < kVarStages - 1 && s2 < nslab; ++s2) issue(s2);
  double acc[4][2];
#pragma unroll
  for (int q = 0; q < 4; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
  for (int ks = 0; ks < nslab; ++ks) {
    if (ks > 0) __syncthreads();             // slab ks-1 consumed by every warp: its stage may be refilled
    if (tid == 0 && ks + kVarStages - 1 < nslab) issue(ks + kVarStages - 1);
    if (warp < nmt) {
      mbar_wait(full_bar + ks % kVarStages, (ks / kVarStages) & 1);
      const double* stg = base + (ks % kVarStages) * kVarTmaStageDoubles;
      const double* Ar = stg + (warp * 8 + fr) * 16;
      const double* Br = stg + 4 * abox + fr * 16;
#pragma unroll
      for (int q = 0; q < kVarBK / 16; ++q)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int co = (((hh * 4 + fk) ^ fr) * 2);      // swizzled 16-byte chunk, in doubles
          const double2 av = *reinterpret_cast<const double2*>(Ar + q * abox + co);
          const double2 bv = *reinterpret_cast<const double2*>(Br + q * kVarCols * 16 + co);
          const int c = hh * 2;
          dmma_8x8x4(acc[c][0], acc[c][1], av.x, bv.x);
          dmma_8x8x4(acc[c + 1][0], acc[c + 1][1], av.y, bv.y);
        }
    }
  }
  __syncthreads();                           // nobody still polls the barriers (re-initialised by the next call)
  if (warp < nmt) {
    double rs = 0.0;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const double w = (acc[0][e] + acc[1][e]) + (acc[2][e] + acc[3][e]);
      rs = fma(w, w, rs);
    }
    rs += __shfl_xor_sync(0xffffffffu, rs, 1);
    rs += __shfl_xor_sync(0xffffffffu, rs, 2);
    if (fk == 0) a.part_rs[(size_t)b * a.mpad + m0 + warp * 8 + fr] = rs;
  }
}

__device__ __forceinline__ void var_small_dispatch(const ScoreArgs& a, int b, int tile, double* smem_raw) {
  if (a.use_tma) var_small_block_tma(a, b, tile, smem_raw);
  else var_small_block(a, b, tile, smem_raw);
}

// EIGHT lanes per candidate m (lane group p = 0..7 sums partials p, p + 8, ... then a fixed shuffle tree):
// deterministic, and a 25-candidate batch finalises in one pass of 200 threads.
template <bool WITH_LINF, bool GENERIC = true>
__device__ __forceinline__ void small_finalize_8(const ScoreArgs& a, int m, int p, bool active, int& clamped) {
  const int nvb = a.np / kVarCols, nmb = a.np / 64;
  double rs = 0.0, mean = 0.0, dist = INFINITY;
  if (active) {
    for (int s = p; s < nvb; s += 8) rs += a.part_rs[(size_t)s * a.mpad + m];
    for (int s = p; s < nmb; s += 8) {
      mean += a.part_mu[(size_t)s * a.mpad + m];
      if (WITH_LINF) dist = fmin(dist, a.part_linf[(size_t)s * a.mpad + m]);
    }
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    rs += __shfl_xor_sync(0xffffffffu, rs, o);
    mean += __shfl_xor_sync(0xffffffffu, mean, o);
    if (WITH_LINF) dist = fmin(dist, __shfl_xor_sync(0xffffffffu, dist, o));
  }
  if (active && p == 0) emit_score<GENERIC>(a, m, rs, mean, dist, clamped);
}

// Host side (score.cu).  The argument block of the scoring kernels for M candidates on `h`; fn: the acquisition
// function (nullptr: UCB with acq->ucb_coefficient).
void fill_score_args(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq, const AcqFn* fn,
                     double* score, double* mu, double* sigma, double* linf, ScoreArgs* pa);
// Argument block + workspaces of the small-pool path.
int prepare_small_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                        double* score, double* mu, double* sigma, double* linf, ScoreArgs* a, bool* with_linf,
                        const AcqFn* fn = nullptr);
size_t cross_small_smem_bytes(int dc, int dk);
size_t var_small_smem_bytes();

}  // namespace vzgp
