// Fused posterior mean/variance + UCB + trust-region scoring over a candidate pool, the
// Philox candidate generator and top-k selection.
//
// Replaces (reference): BayesianScoringFunction.score_with_aux
// (vizier/_src/algorithms/designers/gp/acquisitions.py:177-207) = predict_with_aux
// (stochastic_process_model.py:800-868, TFP posterior_predictive) + UCB (:213-225) +
// _apply_trust_region (:152-174) + TrustRegion.min_linf_distance (:779-820); the candidate
// source of RandomVectorizedStrategy (random_vectorized_optimizer.py:78-100) and the top-k
// bookkeeping of vectorized_base.py:544-587.
//
// One persistent CTA per SM walks 64-candidate tiles:
//   phase 1  K* tile [64 x np] = Matern(x*, X) built 64 columns at a time from shared-memory
//            staged rows (without the trust-region distance, d2 = |a_c|^2 + |b_c|^2 - 2 a_c.b_c of centred
//            features, the cross term on the DMMA pipe); mu = K* alpha and the L-inf trust-region distance
//            are reduced on the fly; each 64-column step of the tile is written to shared memory in the layout of phase 2's
//            TMA boxes and leaves by TMA store to a CTA-private scratch (L2 resident, never re-read by others).
//   phase 2  W = K* . Linv^T in 64 x 128 blocks on the FP64 tensor pipe (mma.sync m16n8k8 f64: on the
//            H100 the m8n8k4 shape issues at half the rate), operands streamed by a TMA producer warp
//            (cp.async.bulk.tensor, 128-byte swizzle) through a 4-stage ring with full/empty mbarriers,
//            exploiting that Linv is lower triangular (k <= j, all-zero fragments skipped); each block
//            is squared and row-summed in registers, W is never stored.  Large pools run in 2-CTA
//            clusters that multicast each Linv box to both CTAs.
//            Eight math warps (2 (M) x 4 (N), a 32 x 32 block each) and the producer warp: 288 threads.
//            One SM sub-partition holds 3 of the 9 warps, which caps the kernel at 168 registers; the
//            64 accumulator registers of a warp tile fit without spills because K* is stored in row-pair
//            order (no register moves to form the A fragments) and the k-group loop is not unrolled.
//   epilogue var = sf2 + sn2 - sum W^2 (clamped at 0), sigma, UCB, trust region, outputs.
#include <cuda.h>

#include <climits>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>

#include "launchers.h"
#include "matern_fast.cuh"
#include "pe_ensemble.cuh"
#include "score_small.cuh"
#include "topk_merge.cuh"
#include "tiles.cuh"

namespace vzgp {

using GP1 = GemmCfg<64, 64, 16, 4, 4>;  // phase-1 thread mapping of the trust-region instances: 256 threads, 4x4 outputs each
constexpr int kThreads = 256;        // consumer threads (8 math warps)
constexpr int kBlockThreads = 288;   // + one TMA producer warp
static_assert(GP1::kThreads == kThreads, "phase 1 maps one d2 block to every math thread");

// Phase-2 tiling: 64 candidates x 128 output columns per pass, k-slabs of 32, 4-stage TMA ring.
// 8 warps as 2 (M) x 4 (N): each warp owns a 32 x 32 block = 2 x 4 m16n8 DMMA tiles.
constexpr int kBN = 128;         // output columns per pass
constexpr int kBK = 32;          // k-slab = 32 columns of K* and Linv
constexpr int kStages = 4;
// K* is stored in row-pair order so that one 16-byte load gives two A-fragment registers in the order
// m16n8k8 wants them.  Pair p of a tile holds rows 16 (p / 8) + p % 8 and that + 8 (rows fr and fr + 8
// of one A fragment); in the scratch each k group of 8 is a dense box of 32 pairs x [8 k][2 rows], and in the
// phase-1 staging pair position 2p + e stands for row pair_row(2p + e).
__host__ __device__ constexpr int pair_pos(int r) { return (((r >> 4) * 8 + (r & 7)) << 1) | ((r >> 3) & 1); }
__host__ __device__ constexpr int pair_row(int pos) { return ((pos >> 4) << 4) + ((pos >> 1) & 7) + ((pos & 1) << 3); }
static_assert(pair_row(pair_pos(13)) == 13 && pair_row(pair_pos(58)) == 58 && pair_pos(8) == 1, "pair order round trip");
// One stage: A box 0..3 | B half0 | B half1, each a dense [rows][16] box written by TMA with the 128-byte
// swizzle (16-byte chunk c of row r lands at chunk c ^ (r & 7)).  A box h: k group h of the slab, 32 row
// pairs x 8 k x 2 rows.  B half: 128 Linv rows x 16 k.
constexpr int kABox = (kTM / 2) * 16;            // doubles
constexpr int kBHalf = kBN * 16;
constexpr int kStageDoubles = 4 * kABox + 2 * kBHalf;   // 6144 doubles = 48 KB
constexpr unsigned kStageBytes = kStageDoubles * sizeof(double);
// Large pools run in clusters of kCluster CTAs on adjacent tiles.  They walk the same slab sequence, so
// every Linv box is loaded from L2 once per cluster: the B operand of a stage is split into kBPieces
// boxes of kBPieceRows rows, and each CTA multicasts its share into the same stage of all of them.
constexpr int kCluster = 2;
constexpr int kBPieces = kCluster < 2 ? 2 : kCluster;
constexpr int kBPieceRows = 2 * kBN / kBPieces;
static_assert(kBPieces % 2 == 0 && kBN % (kBPieces / 2) == 0, "B pieces tile the two halves of a stage");
// Phase 1 aliases the ring: K* staging | candidates [dc][LD] | kTrialBufs x (trials [dc][LD], alpha [64]).
// A staging buffer holds one 64-column step of K* as the eight A boxes that phase 2 loads back, and leaves by
// TMA store.  A 32 KB step's store can take longer than the math of a step at D = 20.  With an L2 persisting
// window on the scratch it did, at about 4 bytes per cycle per SM, which is why k_score installs no window.  So
// the stores get as many staging buffers as fit: three up to dc = 45, two up
// to dc = 61, and above that one, where each step waits for the previous step's store to have read it (one
// more barrier per step).
constexpr int kStgDoubles = 8 * kABox;    // 64 x 64 K* block, 32 KB (a multiple of 1024 bytes: swizzle atoms stay aligned)
constexpr int kTrialBufs = 3;             // trials staged one step ahead, released one step later: one barrier per step
__host__ __device__ constexpr int trial_stride(int dc) { return dc * kLD1 + 64; }
__host__ __device__ constexpr int phase1_doubles(int dc, int nstg) { return nstg * kStgDoubles + dc * kLD1 + kTrialBufs * trial_stride(dc); }
__host__ __device__ constexpr int stg_buffers(int dc) {
  return phase1_doubles(dc, 3) <= kStages * kStageDoubles ? 3 : phase1_doubles(dc, 2) <= kStages * kStageDoubles ? 2 : 1;
}
static_assert(phase1_doubles(kMaxDc, 1) <= kStages * kStageDoubles, "phase-1 staging fits in the ring at every dc");
static_assert(stg_buffers(45) == 3 && stg_buffers(46) == 2 && stg_buffers(61) == 2 && stg_buffers(62) == 1,
              "the staging plan switches at dc = 46 and 62 (tested on both sides)");

#ifdef VZ_SCORE_TIMING
// Instrumented build only (make timing): clock64 sums over all CTAs, read by vzgp_debug_score_timing.
// [0] tiles  [1] phase 1  [2] phase 2  [3] tile gate (barrier after phase 1)  [4] whole tile   (math warp 0)
// [5] math warps waiting on full barriers (summed over the 8 warps)  [6] producer waiting on empty barriers
// phase 1, math warp 0: [7] d2 (the fast instance: n_a + n_b, the DMMA cross term and the categorical terms)  [8] Matern + mu  [9] scratch stores (K* written to the staging buffer, and
// thread 0's TMA store issue)  [10] barriers, cp.async waits and thread 0's waits for the TMA stores
constexpr int kScoreCounters = 11;
__device__ unsigned long long g_score_t[kScoreCounters];
#define VZ_ST(...) __VA_ARGS__
#else
#define VZ_ST(...)
#endif

template <bool WITH_LINF, bool GENERIC>
__global__ void __launch_bounds__(kBlockThreads, 1) k_score(const __grid_constant__ ScoreArgs a) {
  extern __shared__ double smem_raw[];
  // the swizzled TMA boxes need a 1024-byte aligned base
  // (pointer arithmetic on the shared-space pointer so the compiler keeps LDS/STS addressing)
  double* smem = smem_raw + (((1024u - (static_cast<unsigned>(__cvta_generic_to_shared(smem_raw)) & 1023u)) & 1023u) >> 3);
  constexpr int LD = kLD1;
  const int dc = a.kp.dc, dk = a.kp.dk, np = a.np;
  double* ring = smem;                                   // [kStages][kStageDoubles]
  // Without the trust-region distance the features are pre-divided by the length scale (the
  // reference's FeatureScaled form, 2 flops per dimension).  With it, unscaled features are staged
  // so that |a-b| is exact, and the scaling is applied to the squared difference.
  // Phase 1 and phase 2 never overlap in time, so the phase-1 staging buffers alias the ring.
  const int nstg = stg_buffers(dc);
  double* sk = ring;                                     // [nstg][8 boxes]  K* of a step, 1024-byte aligned
  double* sa = sk + nstg * kStgDoubles;                  // [dc][LD]     candidates (transposed)
  double* sb = sa + dc * LD;                             // [3][trial_stride]  trials [dc][LD] and alpha [64]
  double* s_mu = ring + kStages * kStageDoubles;         // [4][64]  one partial mean per column quarter (one [64] with WITH_LINF)
  double* s_linf = s_mu + 256;                           // [64]
  double* s_rowsq = s_linf + 64;                         // [4][64]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_rowsq + 256);  // [kStages] TMA bytes landed
  uint64_t* empty_bar = full_bar + kStages;                         // [kStages] all 8 math warps of every CTA in the cluster released the stage
  int32_t* za = reinterpret_cast<int32_t*>(full_bar + 8);  // [dk][LD]
  int32_t* zb = za + dk * LD;                            // [dk][LD]
  uint8_t* s_mask = reinterpret_cast<uint8_t*>(zb + dk * LD);  // [kMaxDc]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ty = tid / 16, tx = tid % 16;      // phase-1 mapping (16 x 16 threads)
  // Warp grid 2 (M) x 4 (N) of phase 2 (and of the fast instance's phase 1).  Warp w runs on SM sub-partition
  // w % 4, and column quarter wn of a 128-column block runs 4 jb + wn + 1 slabs (Linv is triangular).  Warps
  // 4-7 take quarters 3, 3, 2, 2, so every sub-partition holds quarters {0, 3} or {1, 2}: 8 jb + 5 slab-units
  // per block on each (with wn = warp / 2 it was 8 jb + 4 on two of them and 8 jb + 6 on the other two).
  const int wm = warp & 1, wn = (warp >> 1) ^ (warp >> 2);
  const int fr = lane >> 2, fk = lane & 3;     // fragment row / k within a DMMA tile
  // Linv row (output column) that B fragment row fr stands for within its 8-row group.  An LDS.128 is
  // served 8 lanes at a time; lanes 0-7 are fragment rows 0 and 1.  With the 128-byte swizzle rows r and
  // r^1 keep their chunks in the same 64-byte half, a 2-way bank conflict on every operand load; rows r
  // and r^4 land in opposite halves.  So fr = 2i, 2i+1 read rows i, i+4.  Row sums do not care which
  // column a fragment row holds.  (A, in pair order, reads even and odd chunks and needs no remapping.)
  const int pr = ((fr & 1) << 2) | (fr >> 1);
  // The K* scratch of this CTA is a run of dense 4 KB boxes, one per 8-wide k group g (32 row pairs x 8 k x 2 rows),
  // at box row (blockIdx.x * np / 8 + g) * 32 of mapA: a step's 32 KB and a slab's 16 KB are contiguous in memory.
  auto scratch_box_row = [&](int g) { return ((int)blockIdx.x * (np / 8) + g) * (kTM / 2); };
  // Cluster of ncta CTAs (1 for medium pools, which split a tile's blocks between CTAs, else kCluster).
  // The peers write into this CTA's ring and arrive on its empty barriers, so every gate that keeps the
  // ring or the barriers untouched is cluster-wide when ncta > 1.
  const unsigned crank = cluster_ctarank(), ncta = cluster_nctarank();
  auto tile_gate = [&]() { if (ncta > 1) cluster_sync(); else __syncthreads(); };
  if (tid < kMaxDc) s_mask[tid] = a.tr.mask[tid];
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, ncta * (kThreads / 32)); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  tile_gate();   // barriers initialised in every CTA before any peer multicasts or arrives
  int clamped = 0;
  unsigned slab_n = 0;   // slabs issued (producer) / consumed (math warps) since kernel start: ring position and phase
  const bool is_producer = warp == kThreads / 32;
  auto consumer_sync = [&]() { asm volatile("bar.sync 1, %0;\n" ::"n"(kThreads) : "memory"); };
  // Counters: sums over the tiles that hold candidates (the all-padding tile of a last round is left out).
  VZ_ST(long long t_p1 = 0, t_gate = 0, t_p2 = 0, t_tile = 0, t_wait = 0, w_tile = 0, n_tiles = 0;)
  VZ_ST(long long t_d2 = 0, t_mat = 0, t_st = 0, t_sync = 0;)

  const int ntiles = (a.M + kTM - 1) / kTM;
  const int nblocks = (np + kBN - 1) / kBN;
  const int nsplit = a.nsplit;
  const double* XTu = a.XT + xt_plane(1, dc, np);   // unscaled (trust-region instances)
  const double* XTc = a.XT + xt_plane(2, dc, np);   // centred and scaled (fast instance)
  const double* nb_g = a.XT + xt_norms(dc, np);     // [np] their squared norms
  const double* ctr = a.XT + xt_centre(dc, np);     // [dc] the centre

  // The CTAs of a cluster take adjacent work items and run the same number of rounds.  In the last
  // round a CTA can be left without a tile (work >= ntiles, nsplit == 1): it scores an all-padding tile
  // (m0 >= M, nothing emitted) so that its Linv pieces and stage releases still reach its peers.
  for (int w0 = blockIdx.x - crank; w0 < ntiles * nsplit; w0 += gridDim.x) {
    const int work = w0 + crank;
    const int tile = work / nsplit, split = work - tile * nsplit;
    const int m0 = tile * kTM;
    // Work split of this tile's phase 2 (identical for producer and consumers).
    const int nq = (nsplit == 1) ? nblocks : ((split == nblocks - 1 - split) ? 1 : 2);
    auto block_of = [&](int q) { return (nsplit == 1) ? q : (q == 0 ? split : nblocks - 1 - split); };
    auto slabs_in = [&](int jb) { int kend = (jb + 1) * kBN; if (kend > np) kend = np; return kend / kBK; };
    if (is_producer) {
      // ---- TMA producer warp: waits for phase 1 of this tile, then streams every slab of the
      // tile through the ring, gated only by the per-stage empty barriers.  The gate also waits for
      // phase 1 of the peers: their phase-1 staging aliases the ring this producer multicasts into.
      tile_gate();
      VZ_ST(w_tile = 0;)
      if (lane == 0) {
        const uint16_t cmask = (uint16_t)((1u << ncta) - 1u);
        for (int q = 0; q < nq; ++q) {
          const int jb = block_of(q), nsl = slabs_in(jb);
          for (int ks = 0; ks < nsl; ++ks) {
            const int stage = slab_n % kStages;
            VZ_ST(const long long t0 = clock64();)
            mbar_wait(empty_bar + stage, ((slab_n / kStages) & 1) ^ 1);
            VZ_ST(w_tile += clock64() - t0;)
            double* base = ring + stage * kStageDoubles;
            const int k0 = ks * kBK;
            mbar_expect_tx(full_bar + stage, kStageBytes);   // own A boxes + the B pieces of every CTA
            for (int h = 0; h < 4; ++h)
              tma_load_2d(base + h * kABox, &a.mapA, 0, scratch_box_row(k0 / 8 + h), full_bar + stage);
            for (int p = (int)crank; p < kBPieces; p += (int)ncta) {   // rows >= np: zero fill
              const int half = p / (kBPieces / 2), r0 = (p % (kBPieces / 2)) * kBPieceRows;
              double* dst = base + 4 * kABox + half * kBHalf + r0 * 16;
              if (ncta > 1) tma_load_2d_multicast(dst, &a.mapB, k0 + 16 * half, jb * kBN + r0, full_bar + stage, cmask);
              else tma_load_2d(dst, &a.mapB, k0 + 16 * half, jb * kBN + r0, full_bar + stage);
            }
            ++slab_n;
          }
        }
      }
      __syncwarp();
      VZ_ST(if (m0 < a.M) t_wait += w_tile;)
      continue;
    }
    VZ_ST(const long long t_tile0 = clock64(); w_tile = 0;)
    consumer_sync();  // previous tile fully consumed by the math warps (sa, s_mu, s_rowsq, ring)
    // candidate tile, transposed and in pair order.  The fast instance stages -2 a_c, a_c = (x - centre) / ls
    // (the trials' centre, the reference's FeatureScaled scaling), the A operand of the cross term.
    for (int e = tid; e < kTM * dc; e += kThreads) {
      const int r = e / dc, d = e - r * dc;
      const int gr = m0 + r;
      const double v = gr < a.M ? __ldg(a.Xs + (size_t)gr * dc + d) : 0.0;
      sa[d * LD + pair_pos(r)] = WITH_LINF ? v : -2.0 * ((v - ctr[d]) * a.kp.inv_ls_c[d]);
    }
    if (dk > 0) stage_rows_T_i32(a.Zs, a.M, dk, m0, kTM, za, LD, kThreads);

    // ---------------- phase 1: K* tile, mean, trust-region distance ----------------
    // Trial rows arrive pre-transposed and pre-scaled (XT), 64 columns per step, through a
    // three-deep cp.async buffer: the copy of block jb+1 overlaps the math of block jb, and the buffer
    // it fills was last read in step jb-2, which every thread left before the barrier of step jb-1.
    auto stage_trials = [&](int jb, int buf) {
      double* dst = sb + buf * trial_stride(dc);
      const double* src = WITH_LINF ? XTu : XTc;
      for (int c = tid; c < dc * 32; c += kThreads) {       // dc rows x 32 chunks of 16 B
        const int d = c >> 5, q = c & 31;
        cp_async16(dst + d * LD + q * 2, src + (size_t)d * np + jb * 64 + q * 2, true);
      }
      if (tid < 32) cp_async16(dst + dc * LD + tid * 2, a.alpha + jb * 64 + tid * 2, true);
    };
    // K* of step jb leaves as eight boxes of the scratch's tensor map (mapA, the one phase 2 loads with).
    auto store_step = [&](int jb) {
      const double* src = sk + (jb % nstg) * kStgDoubles;
#pragma unroll 1
      for (int h = 0; h < 8; ++h) tma_store_2d(&a.mapA, 0, scratch_box_row(8 * jb + h), src + h * kABox);
      bulk_commit();
    };
    double mu_part[4], lmin[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { mu_part[i] = 0.0; lmin[i] = INFINITY; }
    const int nj = np / 64;
    stage_trials(0, 0);
    cp_async_commit();
    for (int jb = 0; jb < nj; ++jb) {
      VZ_ST(long long tc = clock64();)
      const int buf = jb % kTrialBufs;
      if (jb + 1 < nj) stage_trials(jb + 1, (jb + 1) % kTrialBufs);
      cp_async_commit();
      // |b_c|^2 of the lane's four columns (fast instance), loaded before the barrier wait
      double2 nbv[2];
      if constexpr (!WITH_LINF) {
#pragma unroll
        for (int nf = 0; nf < 2; ++nf) nbv[nf] = __ldg(reinterpret_cast<const double2*>(nb_g + jb * 64 + 16 * wn + 8 * nf + 2 * fk));
      }
      cp_async_wait<1>();
      // With nstg >= 2 staging buffers, step jb writes the one the store of step jb-nstg reads.  That store was
      // issued at the start of step jb-nstg+1, and at most the nstg-2 stores issued after it may still be reading;
      // once it is done, the barrier below releases the buffer to every thread.
      if (tid == 0) { if (nstg == 3) bulk_wait_read<1>(); else bulk_wait_read<0>(); }
      // Trials of step jb have landed for every thread; every thread has written (and fenced) its part of step
      // jb-1's K* and is done reading the trial buffer of step jb-1.
      consumer_sync();
      if (dk > 0) {  // categorical rows are rare: staged synchronously
        stage_rows_T_i32(a.Z, np, dk, jb * 64, 64, zb, LD, kThreads);
        consumer_sync();
      }
      VZ_ST(t_sync += clock64() - tc; tc = clock64();)
      if (jb > 0 && tid == 0) store_step(jb - 1);
      VZ_ST(t_st += clock64() - tc; tc = clock64();)
      const double* sbj = sb + buf * trial_stride(dc);
      const double* alj = sbj + dc * LD;
      // kv: the sixteen kernel values of this thread (the two instances map them to the step differently).
      double kv[4][4];
      auto ld2 = [](const double* p) { return *reinterpret_cast<const double2*>(p); };
      if constexpr (WITH_LINF) {
        double d2[4][4], lf[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) { d2[i][j] = 0.0; lf[i][j] = 0.0; }
        // Software-pipelined over d: the LDS.128 operands of dimension d + 1 (and its weight and mask) are loaded
        // while the 32 FP64 operations of dimension d run.  The FMA sequence of every element is unchanged.
        double2 a0 = ld2(sa + GP1::row_of(ty, 0)), a1 = ld2(sa + GP1::row_of(ty, 2));
        double2 b0 = ld2(sbj + GP1::col_of(tx, 0)), b1 = ld2(sbj + GP1::col_of(tx, 2));
        double w_n = a.kp.inv_ls2_c[0];
        bool in_tr_n = s_mask[0] != 0;
        for (int d = 0; d < dc; ++d) {
          const int dn = d + 1 < dc ? d + 1 : d;
          const double2 a0n = ld2(sa + dn * LD + GP1::row_of(ty, 0)), a1n = ld2(sa + dn * LD + GP1::row_of(ty, 2));
          const double2 b0n = ld2(sbj + dn * LD + GP1::col_of(tx, 0)), b1n = ld2(sbj + dn * LD + GP1::col_of(tx, 2));
          const double aa[4] = {a0.x, a0.y, a1.x, a1.y}, bb[4] = {b0.x, b0.y, b1.x, b1.y};
          a0 = a0n; a1 = a1n; b0 = b0n; b1 = b1n;
          const double w = w_n;
          const bool in_tr = in_tr_n;
          w_n = a.kp.inv_ls2_c[dn];
          in_tr_n = s_mask[dn] != 0;
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const double df = aa[i] - bb[j];
              d2[i][j] = fma(df * df, w, d2[i][j]);
              if (in_tr) lf[i][j] = fmax(lf[i][j], fabs(df));
            }
        }
        for (int k = 0; k < dk; ++k) {
          const double w = a.kp.inv_ls2_k[k];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int avz = za[k * LD + pair_row(GP1::row_of(ty, i))];   // za is staged in row order
#pragma unroll
            for (int j = 0; j < 4; ++j) d2[i][j] += (avz != zb[k * LD + GP1::col_of(tx, j)]) ? w : 0.0;
          }
        }
        VZ_ST(t_d2 += clock64() - tc; tc = clock64();)
        // The L-inf distances are folded before the Matern block so that they are not live across it.
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if ((jb * 64 + GP1::col_of(tx, j)) < a.tr.rows) lmin[i] = fmin(lmin[i], lf[i][j]);
        // The sixteen kernel values as one straight-line block of the branch-free Matern (independent chains
        // the scheduler can interleave); columns at or past n_valid are zeroed by a select.
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) kv[i][j] = matern52_fast(d2[i][j], a.kp.sf2);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int cj = GP1::col_of(tx, j);
            kv[i][j] = (jb * 64 + cj) < a.n_valid ? kv[i][j] : 0.0;
            mu_part[i] = fma(kv[i][j], alj[cj], mu_part[i]);
          }
        VZ_ST(t_mat += clock64() - tc; tc = clock64();)
      } else {
        // d2 = |a_c|^2 + |b_c|^2 - 2 a_c.b_c of the centred features, the cross term on the DMMA pipe: the warp's
        // 32 x 16 region of the step is 2 x 2 m16n8 tiles whose accumulators start at n_a + n_b.  k slots fk and
        // fk + 4 of k step ks are dimensions 8 ks + 2 fk and 8 ks + 2 fk + 1, the same on both operands (the A loads
        // are LDS.128 of a row pair, the B loads LDS.64; with LD = 66 both are conflict-free).  Dimensions past dc
        // are zero on both sides.  kv[2 mf + f][2 nf + c]: row 32 wm + 16 mf + 8 f + fr, column 16 wn + 8 nf + 2 fk + c.
        const double* Ab = sa + 32 * wm + 2 * fr;   // pair (2 wm + mf) * 8 + fr: rows fr and fr + 8 of M fragment mf
        const double* Bb = sbj + 16 * wn + fr;
        // n_a of the lane's four rows, kept in this warp's slice of s_mu (free until the tile's partial means)
        double* s_na = s_mu + wn * 64 + 32 * wm + fr;
        if (jb == 0) {   // the staged -2 a_c squared and summed, times 1/4 (exact)
          double na[4] = {0.0, 0.0, 0.0, 0.0};
          for (int d = 0; d < dc; ++d)
#pragma unroll
            for (int mf = 0; mf < 2; ++mf) {
              const double2 v = ld2(Ab + d * LD + 16 * mf);
              na[2 * mf] = fma(v.x, v.x, na[2 * mf]);
              na[2 * mf + 1] = fma(v.y, v.y, na[2 * mf + 1]);
            }
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (fk == 0) s_na[8 * i] = 0.25 * na[i];
          __syncwarp();
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int nf = 0; nf < 2; ++nf) { kv[i][2 * nf] = s_na[8 * i] + nbv[nf].x; kv[i][2 * nf + 1] = s_na[8 * i] + nbv[nf].y; }
        auto frag = [&](int ks, double2 (&fa)[2][2], double (&fb)[2][2]) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int d = 8 * ks + 2 * fk + e;
            const bool ok = d < dc;
#pragma unroll
            for (int mf = 0; mf < 2; ++mf) fa[e][mf] = ok ? ld2(Ab + d * LD + 16 * mf) : make_double2(0.0, 0.0);
#pragma unroll
            for (int nf = 0; nf < 2; ++nf) fb[e][nf] = ok ? Bb[d * LD + 8 * nf] : 0.0;
          }
        };
        double2 fa[2][2];
        double fb[2][2];
        frag(0, fa, fb);
        // A remainder of 1-4 dimensions takes one m16n8k4 step instead of a half-empty m16n8k8 one.
        const int k4 = (dc & 7) != 0 && (dc & 7) <= 4, kc = k4 ? dc >> 3 : (dc + 7) >> 3;
#pragma unroll 1
        for (int ks = 0; ks < kc; ++ks) {   // the fragments of k step ks + 1 load under the DMMAs of ks
          double2 ga[2][2];
          double gb[2][2];
          frag(ks + 1 < kc ? ks + 1 : ks, ga, gb);
#pragma unroll
          for (int mf = 0; mf < 2; ++mf)
#pragma unroll
            for (int nf = 0; nf < 2; ++nf)
              dmma_16x8x8(kv[2 * mf][2 * nf], kv[2 * mf][2 * nf + 1], kv[2 * mf + 1][2 * nf], kv[2 * mf + 1][2 * nf + 1],
                          fa[0][mf].x, fa[0][mf].y, fa[1][mf].x, fa[1][mf].y, fb[0][nf], fb[1][nf]);
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int q = 0; q < 2; ++q) { fa[e][q] = ga[e][q]; fb[e][q] = gb[e][q]; }
        }
        if (k4) {   // k slot fk is dimension 8 kc + fk
          const int d = 8 * kc + fk;
          const bool ok = d < dc;
#pragma unroll
          for (int mf = 0; mf < 2; ++mf) {
            const double2 av = ok ? ld2(Ab + d * LD + 16 * mf) : make_double2(0.0, 0.0);
#pragma unroll
            for (int nf = 0; nf < 2; ++nf)
              dmma_16x8x4(kv[2 * mf][2 * nf], kv[2 * mf][2 * nf + 1], kv[2 * mf + 1][2 * nf], kv[2 * mf + 1][2 * nf + 1],
                          av.x, av.y, ok ? Bb[d * LD + 8 * nf] : 0.0);
          }
        }
        for (int k = 0; k < dk; ++k) {
          const double w = a.kp.inv_ls2_k[k];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int avz = za[k * LD + 32 * wm + 8 * i + fr];   // za is staged in row order
#pragma unroll
            for (int j = 0; j < 4; ++j) kv[i][j] += (avz != zb[k * LD + 16 * wn + 8 * (j >> 1) + 2 * fk + (j & 1)]) ? w : 0.0;
          }
        }
        // Instrumented build: wait for the last DMMA's result, so that the d2 counter covers the cross term.
        VZ_ST(if (kv[3][3] == -1.0) t_d2 += 1;)
        VZ_ST(t_d2 += clock64() - tc; tc = clock64();)
        // Rounding can leave d2 a few ulps of n_a + n_b below zero where a candidate is a trial.  matern52_fast needs
        // no clamp for that: 5 d2 < 1e-100 selects s = 0, so k = sf2 exactly as at d2 = 0, while a NaN (a non-finite
        // candidate feature) stays a NaN, as in the difference-first form.
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) kv[i][j] = matern52_fast(kv[i][j], a.kp.sf2);
#pragma unroll
        for (int nf = 0; nf < 2; ++nf) {
          const int cj = 16 * wn + 8 * nf + 2 * fk;
          const double2 al = ld2(alj + cj);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            kv[i][2 * nf] = (jb * 64 + cj) < a.n_valid ? kv[i][2 * nf] : 0.0;
            kv[i][2 * nf + 1] = (jb * 64 + cj + 1) < a.n_valid ? kv[i][2 * nf + 1] : 0.0;
            mu_part[i] = fma(kv[i][2 * nf], al.x, mu_part[i]);
            mu_part[i] = fma(kv[i][2 * nf + 1], al.y, mu_part[i]);
          }
        }
        VZ_ST(t_mat += clock64() - tc; tc = clock64();)
      }
      if (nstg == 1) {   // the single staging buffer: the store of step jb-1 must have read it
        if (tid == 0) bulk_wait_read<0>();
        consumer_sync();
      }
      VZ_ST(t_sync += clock64() - tc; tc = clock64();)
      if constexpr (WITH_LINF) {
        // Rows i = 2 ip, 2 ip + 1 of this thread are pair p = 16 ip + ty: one 16-byte store per column, into chunk
        // c = col % 8 of row p of box col / 8, swizzled to chunk c ^ (p % 8).  A 16-byte store is served 8 lanes at
        // a time, lanes tx = 0-7 of one ty: tx 0-3 and 4-7 write the same chunks of two boxes (4 KB apart, the same
        // banks), so lanes with tx >= 4 take their two columns of a chunk pair in swapped order, filling the odd
        // chunks while tx 0-3 fill the even ones.
        {
          double* stg = sk + (jb % nstg) * kStgDoubles;
          const bool swap = (tx & 4) != 0;
#pragma unroll
          for (int ip = 0; ip < 2; ++ip) {
            const int p = 16 * ip + ty;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = jj ^ 1;
              const double v0 = swap ? kv[2 * ip][j] : kv[2 * ip][jj], v1 = swap ? kv[2 * ip + 1][j] : kv[2 * ip + 1][jj];
              const int cj = GP1::col_of(tx, jj) ^ (swap ? 1 : 0);
              *reinterpret_cast<double2*>(stg + (cj >> 3) * kABox + p * 16 + (((cj & 7) ^ (p & 7)) * 2)) = make_double2(v0, v1);
            }
          }
        }
      } else {
        // Rows fr and fr + 8 of M fragment mf are pair p = (2 wm + mf) * 8 + fr, and column 2 fk + c of N fragment nf
        // is chunk 2 fk + c of row p of box 2 wn + nf, swizzled to chunk (2 fk + c) ^ fr.  The 8 lanes of a 16-byte
        // store phase (fr = 2i, 2i + 1) fill the even chunks of one row and the odd ones of the next: no conflict.
        double* stg = sk + (jb % nstg) * kStgDoubles;
#pragma unroll
        for (int mf = 0; mf < 2; ++mf) {
          const int p = (2 * wm + mf) * 8 + fr;
#pragma unroll
          for (int nf = 0; nf < 2; ++nf)
#pragma unroll
            for (int c = 0; c < 2; ++c)
              *reinterpret_cast<double2*>(stg + (2 * wn + nf) * kABox + p * 16 + (((2 * fk + c) ^ fr) * 2)) =
                  make_double2(kv[2 * mf][2 * nf + c], kv[2 * mf + 1][2 * nf + c]);
        }
      }
      fence_proxy_async_smem();   // these writes before the TMA store that reads them (issued after the next barrier)
      VZ_ST(t_st += clock64() - tc;)
    }
    // The staging writes of the last step are done everywhere; its store goes out, and every K* store of the
    // tile is complete (written to global memory) before the tile gate.  The gate's barrier then orders them
    // before the producer's TMA loads of the tile in phase 2: both are async-proxy accesses to global memory,
    // so completion of the bulk group, followed by the barrier, is all the ordering the loads need.
    VZ_ST(long long tc = clock64();)
    consumer_sync();
    VZ_ST(t_sync += clock64() - tc; tc = clock64();)
    if (tid == 0) store_step(nj - 1);
    VZ_ST(t_st += clock64() - tc; tc = clock64();)
    if (tid == 0) bulk_wait<0>();
    VZ_ST(t_sync += clock64() - tc;)
    cp_async_wait<0>();
    if constexpr (WITH_LINF) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
          mu_part[i] += __shfl_xor_sync(0xffffffffu, mu_part[i], o);
          lmin[i] = fmin(lmin[i], __shfl_xor_sync(0xffffffffu, lmin[i], o));
        }
        if (tx == 0) {
          s_mu[pair_row(GP1::row_of(ty, i))] = mu_part[i];
          s_linf[pair_row(GP1::row_of(ty, i))] = lmin[i];
        }
      }
    } else {   // the four lanes of a fragment row, then the four column quarters in the epilogue
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        mu_part[i] += __shfl_xor_sync(0xffffffffu, mu_part[i], 1);
        mu_part[i] += __shfl_xor_sync(0xffffffffu, mu_part[i], 2);
        if (fk == 0) s_mu[wn * 64 + 32 * wm + 8 * i + fr] = mu_part[i];
      }
      if (tid < kTM) s_linf[tid] = INFINITY;
    }
    fence_proxy_async();  // generic-proxy writes (scratch tile, aliased smem) before async-proxy (TMA) accesses
    VZ_ST(const long long t1 = clock64();)
    tile_gate();          // this CTA's scratch tile is complete and visible; the peers are done with their staging
    VZ_ST(const long long t2 = clock64();)

    // ---------------- phase 2: row sums of (K* Linv^T)^2 on the DMMA pipe ----------------
    // Slab (jb, ks): A = K*[0:64, ks*32 : +32] (four pair-order boxes), B = Linv[jb*128 : +128, ks*32 : +32];
    // block jb needs ks < min(np, (jb+1)*128)/32 because Linv is lower triangular.  The slab
    // stream is flattened over blocks so the TMA ring never drains between blocks.
    // With nsplit > 1 this CTA takes blocks {split, nblocks-1-split} (balanced triangular work).
    // acc[mf][f][g][c]: M fragment mf (tile rows wm*32 + mf*16 + ...), fragment row fr + 8f, column fragment g.
    double rowsq[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    for (int q = 0; q < nq; ++q) {
      const int jb = block_of(q);
      double acc[2][2][4][2];
#pragma unroll
      for (int mf = 0; mf < 2; ++mf)
#pragma unroll
        for (int f = 0; f < 2; ++f)
#pragma unroll
          for (int g = 0; g < 4; ++g) { acc[mf][f][g][0] = 0.0; acc[mf][f][g][1] = 0.0; }
      const int nsl = slabs_in(jb);
      const int col_base = jb * kBN + wn * 32;   // first output column of this warp
      for (int ks = 0; ks < nsl; ++ks) {
        const int stage = slab_n % kStages;
        VZ_ST(const long long tw = clock64();)
        mbar_wait(full_bar + stage, (slab_n / kStages) & 1);   // TMA bytes of this slab have landed
        VZ_ST(w_tile += clock64() - tw;)
        ++slab_n;
        // Fragment loads are 16 bytes: lane (fr, fk) takes k = 8h + 2fk and 8h + 2fk + 1 of each
        // 8-wide k group h as the k slots fk and fk + 4 of one m16n8k8 (the k order inside a slab is
        // irrelevant as long as A and B agree).  A: one load per k gives rows fr and fr + 8 of M fragment
        // mf (pair row (wm*2 + mf)*8 + fr of box h, chunk k % 8), i.e. a0, a1 or a2, a3 in register order.
        // B: one load gives both k of column fr, which reads Linv row ... + pr.  Every row base is a
        // multiple of 8, so the swizzle XOR is fr for A and pr for B; both are conflict-free.
        const double* stg = ring + stage * kStageDoubles;
        const double* Arow0 = stg + (wm * 16 + fr) * 16;            // + h*kABox + mf*8*16 + chunk*2
        const double* Brow0 = stg + 4 * kABox + (wn * 32 + pr) * 16;
        const int k0 = ks * kBK;
        // Linv[c, k] = 0 for k > c.  k0 and col_base are multiples of 32: slabs right of this
        // warp's 32 columns contribute nothing; in the diagonal slab (k0 == col_base) the k group
        // h only reaches column fragments g >= h.
        // k group h of the slab: 4 B and 4 A fragment loads, then 8 DMMAs (fewer in the diagonal slab).
        auto group = [&](int h, bool diag) {
          const int co = ((((h & 1) * 4 + fk) ^ pr) * 2);   // swizzled 16-byte B chunk, in doubles
          auto live = [&](int g) { return !(diag && g < h); };   // columns of fragment g < h lie left of k group h
          double2 b[4];
#pragma unroll
          for (int g = 0; g < 4; ++g)
            if (live(g)) b[g] = *reinterpret_cast<const double2*>(Brow0 + (h >> 1) * kBHalf + g * 8 * 16 + co);
#pragma unroll
          for (int mf = 0; mf < 2; ++mf) {
            const double* Ah = Arow0 + h * kABox + mf * 8 * 16;
            const double2 a01 = *reinterpret_cast<const double2*>(Ah + (((2 * fk) ^ fr) * 2));       // k = 8h + 2fk
            const double2 a23 = *reinterpret_cast<const double2*>(Ah + (((2 * fk + 1) ^ fr) * 2));   // k = 8h + 2fk + 1
#pragma unroll
            for (int g = 0; g < 4; ++g)
              if (live(g))
                dmma_16x8x8(acc[mf][0][g][0], acc[mf][0][g][1], acc[mf][1][g][0], acc[mf][1][g][1],
                            a01.x, a01.y, a23.x, a23.y, b[g].x, b[g].y);
          }
        };
        // The group loops are not unrolled: unrolled, ptxas hoists the loads of all four groups and runs
        // out of registers.  A group's eight DMMAs keep the pipe busy while the other warp of the SM
        // sub-partition waits for its loads.  The full slab has no predicate; the diagonal slab (one in
        // every nsl of a warp) predicates its DMMAs on g >= h.
        if (k0 < col_base) {
#pragma unroll 1
          for (int h = 0; h < 4; ++h) group(h, false);
        } else if (k0 == col_base) {
#pragma unroll 1
          for (int h = 0; h < 4; ++h) group(h, true);
        }
        __syncwarp();
        if ((unsigned)lane < ncta) mbar_arrive_cluster(empty_bar + stage, lane);   // the stage of every CTA it was multicast into
      }
#pragma unroll
      for (int mf = 0; mf < 2; ++mf)
#pragma unroll
        for (int f = 0; f < 2; ++f)
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            rowsq[mf][f] = fma(acc[mf][f][g][0], acc[mf][f][g][0], rowsq[mf][f]);
            rowsq[mf][f] = fma(acc[mf][f][g][1], acc[mf][f][g][1], rowsq[mf][f]);
          }
    }
    VZ_ST(const long long t3 = clock64();)
    cp_async_wait<0>();
    // combine the 4 lanes that share a fragment row, then the four N-warps through smem
#pragma unroll
    for (int mf = 0; mf < 2; ++mf)
#pragma unroll
      for (int f = 0; f < 2; ++f) {
        rowsq[mf][f] += __shfl_xor_sync(0xffffffffu, rowsq[mf][f], 1);
        rowsq[mf][f] += __shfl_xor_sync(0xffffffffu, rowsq[mf][f], 2);
        if (fk == 0) s_rowsq[wn * 64 + wm * 32 + mf * 16 + f * 8 + fr] = rowsq[mf][f];
      }
    consumer_sync();
    // ---------------- epilogue ----------------
    if (tid < kTM) {
      const int r = tid, m = m0 + r;
      if (m < a.M) {
        const double rs = (s_rowsq[r] + s_rowsq[64 + r]) + (s_rowsq[128 + r] + s_rowsq[192 + r]);
        const double mu = WITH_LINF ? s_mu[r] : (s_mu[r] + s_mu[64 + r]) + (s_mu[128 + r] + s_mu[192 + r]);
        if (nsplit == 1) {
          emit_score<GENERIC>(a, m, rs, mu, s_linf[r], clamped);
        } else {
          a.part[(size_t)split * a.mpad + m] = rs;
          if (split == 0) {
            a.part[(size_t)nsplit * a.mpad + m] = mu;
            a.part[(size_t)(nsplit + 1) * a.mpad + m] = s_linf[r];
          }
        }
      }
    }
    VZ_ST(if (m0 < a.M) { t_p1 += t1 - t_tile0; t_gate += t2 - t1; t_p2 += t3 - t2; t_tile += clock64() - t_tile0; t_wait += w_tile; ++n_tiles; })
  }
  if (clamped) atomicAdd(a.clamp_count, clamped);
#ifdef VZ_SCORE_TIMING
  if (lane == 0) {
    if (is_producer) {
      atomicAdd(&g_score_t[6], (unsigned long long)t_wait);
    } else {
      atomicAdd(&g_score_t[5], (unsigned long long)t_wait);
      if (warp == 0) {
        atomicAdd(&g_score_t[0], (unsigned long long)n_tiles);
        atomicAdd(&g_score_t[1], (unsigned long long)t_p1);
        atomicAdd(&g_score_t[2], (unsigned long long)t_p2);
        atomicAdd(&g_score_t[3], (unsigned long long)t_gate);
        atomicAdd(&g_score_t[4], (unsigned long long)t_tile);
        atomicAdd(&g_score_t[7], (unsigned long long)t_d2);
        atomicAdd(&g_score_t[8], (unsigned long long)t_mat);
        atomicAdd(&g_score_t[9], (unsigned long long)t_st);
        atomicAdd(&g_score_t[10], (unsigned long long)t_sync);
      }
    }
  }
#endif
  if (ncta > 1) cluster_sync();   // no CTA exits while a peer can still multicast into it or arrive on its barriers
}

// nsplit > 1: sums the partial row sums in a fixed order and emits the scores.  MES: the MaxValueEntropySearch
// instance (the UCB / LCB / EI / PI one keeps its register budget).
template <bool MES>
__global__ void k_score_finalize(const ScoreArgs a) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  int clamped = 0;
  if (m < a.M) {
    double rs = 0.0;
    for (int s = 0; s < a.nsplit; ++s) rs += a.part[(size_t)s * a.mpad + m];
    emit_score<true, MES>(a, m, rs, a.part[(size_t)a.nsplit * a.mpad + m], a.part[(size_t)(a.nsplit + 1) * a.mpad + m],
                          clamped);
  }
  if (clamped) atomicAdd(a.clamp_count, clamped);
}

// Stand-alone kernels of the small-pool path (device functions in score_small.cuh).
template <bool WITH_LINF>
__global__ void __launch_bounds__(kSmallThreads) k_cross_small(const ScoreArgs a) {
  extern __shared__ double smem_raw[];
  cross_small_block<WITH_LINF>(a, blockIdx.x, blockIdx.y >> 2, blockIdx.y & 3, smem_raw);
}
__global__ void __launch_bounds__(kSmallThreads) k_var_small(const __grid_constant__ ScoreArgs a) {
  extern __shared__ double smem_raw[];
  var_small_dispatch(a, blockIdx.x, blockIdx.y, smem_raw);
}
template <bool WITH_LINF, bool MES>
__global__ void __launch_bounds__(256) k_small_finalize(const ScoreArgs a) {
  const int m = blockIdx.x * 32 + (threadIdx.x >> 3);
  int clamped = 0;
  small_finalize_8<WITH_LINF, true, MES>(a, m, threadIdx.x & 7, m < a.M, clamped);
  if (clamped) atomicAdd(a.clamp_count, clamped);
}

size_t cross_small_smem_bytes(int dc, int dk) { return sizeof(double) * 2 * dc * kLD1 + sizeof(int32_t) * 2 * dk * kLD1; }
size_t var_small_smem_bytes() {
  const size_t cp = sizeof(double) * kVarStages * kVarStageDoubles, tma = 1024 + sizeof(double) * kVarStages * kVarTmaStageDoubles;
  return cp > tma ? cp : tma;
}

// ---- host side: TMA descriptors ------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  // function-local static with an initialiser: thread-safe (handles are driven from several host threads)
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    EncodeTiledFn f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      f = reinterpret_cast<EncodeTiledFn>(p);
    cudaGetLastError();
    return f;
  }();
  return fn;
}

// fp64 matrix [rows x cols] with row pitch ld (elements); box = box_rows x 16 doubles, 128-byte swizzle.
static int make_map(CUtensorMap* m, const double* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                    bool l2_promotion = true) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return VZGP_ERR_CUDA; }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * sizeof(double)};
  cuuint32_t box[2] = {16, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  l2_promotion ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return VZGP_ERR_CUDA; }
  return 0;
}

int make_tensor_map_f64(void* map, const double* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  // no L2 promotion: the dataflow kernel loads tiles whose NEIGHBOURS are still being written by other CTAs
  static const bool promo = [] { const char* e = getenv("VZGP_DF_L2PROMO"); return e && e[0] == '1'; }();
  return make_map(static_cast<CUtensorMap*>(map), base, rows, cols, ld, box_rows, promo);
}

int make_tensor_map_u8(void* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                       const uint32_t* box, bool promote_256) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return VZGP_ERR_CUDA; }
  cuuint64_t gdim[3], gstride[2];
  cuuint32_t bx[3], estr[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) gstride[i] = strides[i];
  CUresult r = fn(static_cast<CUtensorMap*>(map), CU_TENSOR_MAP_DATA_TYPE_UINT8, (cuuint32_t)rank, const_cast<void*>(base),
                  gdim, gstride, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  promote_256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (u8) failed with CUresult %d", (int)r); return VZGP_ERR_CUDA; }
  return 0;
}

size_t score_smem_bytes(int dc, int dk, bool with_linf) {
  (void)with_linf; (void)dc;   // phase 1's plan for any dc fits in the ring (stg_buffers)
  return 1024 + sizeof(double) * (kStages * kStageDoubles + 256 + 64 + 256 + 8) +
         sizeof(int32_t) * dk * 2 * kLD1 + kMaxDc;
}

// K* scratch of `bytes` bytes on the handle.  It is written and re-read by the same CTA tile after tile.
// persist: pin it in L2 (persisting access-policy window) so its dirty lines are overwritten in place instead
// of being evicted to HBM; the small-pool route asks for that.  Best effort: failures only cost DRAM write-backs.
// k_score asks for no window and removes one a small-pool call installed: its K* leaves by TMA store, and with
// the window installed those stores drained so slowly that phase 1 waited on them (C2: 2.90 ms per pass against
// 2.77 ms without the window, H100 80GB HBM3, 700 W), while the generic stores it replaced ran at the same speed
// either way.
static int ensure_scratch(vzgp_handle* h, size_t scratch_bytes, bool persist) {
  if (scratch_bytes > h->scratch.bytes) VZ_TRY(h->scratch.reserve(scratch_bytes));
  if (!persist) {
    if (h->scratch_window != nullptr) {
      cudaStreamAttrValue attr;
      memset(&attr, 0, sizeof(attr));   // num_bytes 0: no window
      cudaStreamSetAttribute(h->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
      cudaGetLastError();
      h->scratch_window = nullptr;
    }
    return 0;
  }
  if (h->scratch_window != h->scratch.ptr) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, h->device) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
      size_t want = h->scratch.bytes;
      if (want > (size_t)prop.persistingL2CacheMaxSize) want = (size_t)prop.persistingL2CacheMaxSize;
      cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want);
      cudaStreamAttrValue attr;
      memset(&attr, 0, sizeof(attr));
      size_t win = h->scratch.bytes;
      if (win > (size_t)prop.accessPolicyMaxWindowSize) win = (size_t)prop.accessPolicyMaxWindowSize;
      attr.accessPolicyWindow.base_ptr = h->scratch.ptr;
      attr.accessPolicyWindow.num_bytes = win;
      attr.accessPolicyWindow.hitRatio = win > 0 ? (float)((double)want / (double)win > 1.0 ? 1.0 : (double)want / (double)win) : 0.f;
      attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      cudaStreamSetAttribute(h->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
      cudaGetLastError();
    }
    h->scratch_window = h->scratch.ptr;
  }
  return 0;
}

// Clusters of cfg's shape that fit on the device at once (the GPCs decide it: not every SM count
// divides into clusters).  Cached per device, kernel and shared-memory size.
static int max_active_clusters(const void* kfn, const cudaLaunchConfig_t& cfg, int* out) {
  static std::mutex mu;
  static std::map<std::tuple<int, const void*, size_t>, int> cache;
  int dev = 0;
  VZ_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  int& n = cache[{dev, kfn, cfg.dynamicSmemBytes}];
  if (n == 0) {
    cudaLaunchConfig_t c = cfg;
    c.gridDim = dim3(cfg.attrs[0].val.clusterDim.x);
    VZ_CUDA(cudaOccupancyMaxActiveClusters(&n, kfn, &c));
    if (n <= 0) { set_error("no cluster of the score kernel fits on device %d", dev); return VZGP_ERR_CUDA; }
  }
  *out = n;
  return 0;
}

void fill_score_args(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq, const AcqFn* fn,
                     double* score, double* mu, double* sigma, double* linf, ScoreArgs* pa) {
  ScoreArgs& a = *pa;
  const int ntiles = (M + kTM - 1) / kTM;
  a.Xs = Xs; a.Zs = Zs; a.M = M;
  a.XT = h->XT.as<double>(); a.Z = h->Z.as<int32_t>();
  a.np = h->np; a.n_valid = h->n_valid;
  a.Linv = h->Linv.as<double>(); a.ldi = h->np;
  a.alpha = h->alpha.as<double>();
  a.kp = h->kp; a.sn2 = h->sn2;
  a.acq = acq_fn_of(acq, fn);
  a.tr = trust_region_of(h, *acq, acq->tr_strict);
  a.scratch = h->scratch.as<double>();
  a.mpad = ntiles * kTM;
  a.nsplit = 1;
  a.box_rows = kTM;
  static const int tma_small = [] { const char* e = getenv("VZGP_SMALL_TMA"); return e ? atoi(e) : 1; }();   // 0: cp.async variant
  a.use_tma = tma_small;
  a.part = a.part_rs = a.part_mu = a.part_linf = nullptr;
  a.score = score; a.mu = mu; a.sigma = sigma; a.linf = linf;
  a.clamp_count = h->small.as<int>();  // slot 0
}

int prepare_small_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                        double* score, double* mu, double* sigma, double* linf, ScoreArgs* a, bool* with_linf,
                        const AcqFn* fn) {
  const int ntiles = (M + kTM - 1) / kTM;
  VZ_TRY(ensure_scratch(h, (size_t)ntiles * kTM * h->np * sizeof(double), true));
  fill_score_args(h, Xs, Zs, M, acq, fn, score, mu, sigma, linf, a);
  const int nvb = h->np / kVarCols, nmb = h->np / 64;
  VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)(nvb + 2 * nmb) * a->mpad));
  a->part_rs = h->Tws.as<double>();
  a->part_mu = a->part_rs + (size_t)nvb * a->mpad;
  a->part_linf = a->part_mu + (size_t)nmb * a->mpad;
  *with_linf = (linf != nullptr) || tr_needs_distance(a->tr);
  // TMA boxes of the W phase: K* rows of one tile x 16 doubles, and 8 rows of Linv x 16 doubles.
  a->box_rows = ntiles == 1 ? ((M + 7) / 8) * 8 : kTM;
  VZ_TRY(make_map(&a->mapA, a->scratch, (uint64_t)ntiles * kTM, (uint64_t)h->np, (uint64_t)h->np, (uint32_t)a->box_rows));
  VZ_TRY(make_map(&a->mapB, a->Linv, (uint64_t)h->np, (uint64_t)h->np, (uint64_t)h->np, kVarCols));
  return 0;
}

// ---------------------------------------------------------------------------
// General scoring path: explicit K* and W = K* Linv^T, then one warp per candidate.  Taken by models the
// fused kernels do not cover - today the `linear_coef` variant (tuned_gp_models.py:203-245), whose kernel
// is Matern + feature-scaled linear (so k(x*, x*) is not constant) and whose GP has a constant mean.
// Same results contract as k_score; ~3x the HBM/L2 traffic and DFMA instead of DMMA (k_gemm_nt_tri).
// ---------------------------------------------------------------------------
struct GeneralArgs {
  const double* Xs;      // [mp x dc] padded candidates of this chunk
  const double* Ks;      // [mp x np]
  const double* W;       // [mp x np]
  const double* X;       // [np x dc] trials
  const double* alpha;
  int mc, np, n_valid, dc;
  KernelParams kp;
  double sn2, mean_const;
  AcqFn acq;
  TrustRegion tr;
  int want_linf;
  double* score; double* mu; double* sigma; double* linf;
  int* clamp_count;
};

// One warp per candidate.  MES: the MaxValueEntropySearch instance, its K samples split over lanes 0-7.
template <bool MES>
__global__ void __launch_bounds__(256) k_general_finalize(GeneralArgs a) {
  const int m = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (m >= a.mc) return;
  const double* ks = a.Ks + (size_t)m * a.np;
  const double* w = a.W + (size_t)m * a.np;
  double mean = 0.0, rs = 0.0;
  for (int j = lane; j < a.n_valid; j += 32) mean = fma(ks[j], a.alpha[j], mean);
  for (int j = lane; j < a.np; j += 32) rs = fma(w[j], w[j], rs);
  double dist = a.want_linf ? tr_lane_distance(a.tr, a.Xs + (size_t)m * a.dc, a.X, a.dc, lane) : INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mean += __shfl_xor_sync(0xffffffffu, mean, o);
    rs += __shfl_xor_sync(0xffffffffu, rs, o);
    dist = fmin(dist, __shfl_xor_sync(0xffffffffu, dist, o));
  }
  if (!MES && lane != 0) return;
  double kss = a.kp.sf2;
  if (a.kp.use_linear) {
    double uu = 0.0;
    for (int d = 0; d < a.dc; ++d) {
      const double u = fma(a.Xs[(size_t)m * a.dc + d], a.kp.inv_ls_c[d], -a.kp.lin_b);
      uu = fma(u, u, uu);
    }
    kss = fma(a.kp.lin_a, uu, kss);
  }
  mean += a.mean_const;
  double var = kss - rs + a.sn2;
  if (var < 0.0) { var = 0.0; if (lane == 0) atomicAdd(a.clamp_count, 1); }
  const double sd = sqrt(var);
  double acq;
  if (MES) {
    acq = mes_value_8(a.acq, mean, sd, lane & 7);
    if (lane != 0) return;
  } else {
    acq = acq_value<false>(a.acq, mean, sd);
  }
  a.score[m] = tr_apply(a.tr, acq, dist);
  if (a.mu) a.mu[m] = mean;
  if (a.sigma) a.sigma[m] = sd;
  if (a.linf) a.linf[m] = dist;
}

int general_chunk_buffers(vzgp_handle* h, GeneralChunk* c) {
  const int np = h->np, dc = h->dc, dk = h->dk;
  const size_t nks = (size_t)kGeneralChunk * np, nx = (size_t)kGeneralChunk * (dc > 0 ? dc : 1);
  VZ_TRY(h->gen.reserve(sizeof(double) * (2 * nks + nx) + sizeof(int32_t) * (size_t)kGeneralChunk * (dk > 0 ? dk : 1)));
  c->Ks = h->gen.as<double>();
  c->W = c->Ks + nks;
  c->Xp = c->W + nks;
  c->Zp = reinterpret_cast<int32_t*>(c->Xp + nx);
  return 0;
}

int launch_general_chunk(vzgp_handle* h, const double* Xs, const int32_t* Zs, int mc, const GeneralChunk& c) {
  const int np = h->np, dc = h->dc, dk = h->dk, mp = round_up(mc, 64);
  if (dc > 0) VZ_TRY(launch_pad_rows(h, Xs, mc, dc, mp, c.Xp));
  if (dk > 0) VZ_TRY(launch_pad_rows_i32(h, Zs, mc, dk, mp, c.Zp));
  VZ_TRY(launch_cross_kernel(h, c.Xp, c.Zp, mp, h->X.as<double>(), h->Z.as<int32_t>(), np, h->n_valid, h->kp, c.Ks, np));
  return launch_gemm_nt_tri(h, c.Ks, np, mp, h->Linv.as<double>(), np, np, c.W, np);
}

static int launch_score_general(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                                const AcqFn* fn, double* score, double* mu, double* sigma, double* linf) {
  const int np = h->np, dc = h->dc, dk = h->dk;
  constexpr int kChunk = kGeneralChunk;
  GeneralChunk c;
  VZ_TRY(general_chunk_buffers(h, &c));
  GeneralArgs a;
  a.Ks = c.Ks; a.W = c.W; a.Xs = c.Xp; a.X = h->X.as<double>(); a.alpha = h->alpha.as<double>();
  a.np = np; a.n_valid = h->n_valid; a.dc = dc; a.kp = h->kp; a.sn2 = h->sn2; a.mean_const = h->mean_const;
  a.acq = acq_fn_of(acq, fn);
  a.tr = trust_region_of(h, *acq, acq->tr_strict);
  a.want_linf = (linf != nullptr) || tr_needs_distance(a.tr);
  a.clamp_count = h->small.as<int>();
  for (int m0 = 0; m0 < M; m0 += kChunk) {
    const int mc = M - m0 < kChunk ? M - m0 : kChunk;
    VZ_TRY(launch_general_chunk(h, dc > 0 ? Xs + (size_t)m0 * dc : Xs, dk > 0 ? Zs + (size_t)m0 * dk : Zs, mc, c));
    a.mc = mc;
    a.score = score + m0; a.mu = mu ? mu + m0 : nullptr; a.sigma = sigma ? sigma + m0 : nullptr;
    a.linf = linf ? linf + m0 : nullptr;
    if (a.acq.main.kind == VZGP_ACQ_MES) k_general_finalize<true><<<(mc + 7) / 8, 256, 0, h->stream>>>(a);
    else k_general_finalize<false><<<(mc + 7) / 8, 256, 0, h->stream>>>(a);
    VZ_CHECK_LAUNCH();
    h->launches++;
  }
  return 0;
}

int launch_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                 double* score, double* mu, double* sigma, double* linf, const AcqFn* fn) {
  if (M <= 0) return 0;
  auto record = [&](int route, int nsplit, int grid) { h->score_route = route; h->score_nsplit = nsplit; h->score_grid = grid; };
  // The linear_coef kernel and models past kMaxDk categorical features are scored by the general route only.
  if (h->kp.use_linear || h->dk > kMaxDk) {
    record(VZGP_ROUTE_GENERAL, 0, 0);
    return launch_score_general(h, Xs, Zs, M, acq, fn, score, mu, sigma, linf);
  }
  const int ntiles = (M + kTM - 1) / kTM;
  const int nblocks = (h->np + kBN - 1) / kBN;
  // Pools of a few tiles (acquisition-optimiser batches) take the trial-axis decomposition.
  static const int env_small_tiles = [] {
    const char* e = getenv("VZGP_SMALL_TILES");   // tuning / test hook; 0 disables the small-pool path
    return e ? atoi(e) : 8;
  }();
  const int small_tiles_max = h->small_tiles >= 0 ? h->small_tiles : env_small_tiles;
  ScoreArgs a;
  if (ntiles <= small_tiles_max) {
    record(VZGP_ROUTE_SMALL, 0, 0);
    bool with_linf = false;
    VZ_TRY(prepare_small_score(h, Xs, Zs, M, acq, score, mu, sigma, linf, &a, &with_linf, fn));
    const int nvb = h->np / kVarCols, nmb = h->np / 64;
    const size_t sm1 = cross_small_smem_bytes(h->dc, h->dk), sm2 = var_small_smem_bytes();
    const dim3 g1(nmb, ntiles * 4), g2(nvb, ntiles);
    if (with_linf) {
      VZ_TRY(raise_dyn_smem((const void*)k_cross_small<true>, sm1));
      k_cross_small<true><<<g1, kSmallThreads, sm1, h->stream>>>(a);
    } else {
      VZ_TRY(raise_dyn_smem((const void*)k_cross_small<false>, sm1));
      k_cross_small<false><<<g1, kSmallThreads, sm1, h->stream>>>(a);
    }
    VZ_CHECK_LAUNCH();
    VZ_TRY(raise_dyn_smem((const void*)k_var_small, sm2));
    k_var_small<<<g2, kSmallThreads, sm2, h->stream>>>(a);
    VZ_CHECK_LAUNCH();
    const bool mes = a.acq.main.kind == VZGP_ACQ_MES;
    if (with_linf) (mes ? k_small_finalize<true, true> : k_small_finalize<true, false>)<<<(M + 31) / 32, 256, 0, h->stream>>>(a);
    else (mes ? k_small_finalize<false, true> : k_small_finalize<false, false>)<<<(M + 31) / 32, 256, 0, h->stream>>>(a);
    VZ_CHECK_LAUNCH();
    h->launches += 3;
    return 0;
  }
  {
    // Default off: on the H100 the 28 int8 digit products per fp64 product cost more than the FP64 DMMA pipe
    // (C2 pool: 5.18 ms for k_score_i8 against 4.35 ms for k_score, H100 80GB HBM3 at a 700 W power limit).
    static const int env_i8 = [] { const char* e = getenv("VZGP_SCORE_I8"); return e ? atoi(e) : 0; }();
    const int want = h->score_i8 >= 0 ? h->score_i8 : env_i8;
    if (want && score_i8_eligible(h, M)) {
      record(VZGP_ROUTE_I8, 1, 0);   // launch_score_i8 records its grid
      return launch_score_i8(h, Xs, Zs, M, acq, score, mu, sigma, linf, fn);
    }
  }
  // Medium pools cannot fill the GPU with one CTA per tile: share each tile's output column
  // blocks between nsplit CTAs (each recomputes the cheap K* tile).  Their CTAs walk different
  // block sequences, so they run as clusters of one; large pools run as clusters of kCluster.
  int nsplit = 1;
  if (ntiles * 2 <= h->sm_count && nblocks >= 2) nsplit = (nblocks + 1) / 2;
  const int nwork = ntiles * nsplit;
  const int csize = nsplit == 1 ? kCluster : 1;
  const bool need_linf = (linf != nullptr) || tr_needs_distance(trust_region_of(h, *acq, acq->tr_strict));
  const size_t sm = score_smem_bytes(h->dc, h->dk, need_linf);
  if (sm > 227 * 1024) {
    set_error("score kernel needs %zu bytes of shared memory (Dc=%d with trust-region distance)", sm, h->dc);
    return VZGP_ERR_UNSUPPORTED;
  }
  const bool generic = !acq_fn_is_ucb(acq_fn_of(acq, fn));
  const void* kfn = generic ? (need_linf ? (const void*)k_score<true, true> : (const void*)k_score<false, true>)
                            : (need_linf ? (const void*)k_score<true, false> : (const void*)k_score<false, false>);
  VZ_TRY(raise_dyn_smem(kfn, sm));
  cudaLaunchAttribute cattr[1];
  cattr[0].id = cudaLaunchAttributeClusterDimension;
  cattr[0].val.clusterDim.x = csize; cattr[0].val.clusterDim.y = 1; cattr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(kBlockThreads); cfg.dynamicSmemBytes = sm; cfg.stream = h->stream;
  cfg.attrs = cattr; cfg.numAttrs = 1;
  // Persistent grid: as many clusters as can be co-resident, at most one per csize work items.
  int slots = h->sm_count;
  if (csize > 1) VZ_TRY(max_active_clusters(kfn, cfg, &slots));
  const int want = (nwork + csize - 1) / csize;
  const int grid = (want < slots ? want : slots) * csize;
  cfg.gridDim = dim3(grid);
  record(nsplit > 1 ? VZGP_ROUTE_SPLIT : VZGP_ROUTE_CLUSTER, nsplit, grid);
  VZ_TRY(ensure_scratch(h, (size_t)grid * kTM * h->np * sizeof(double), false));
  fill_score_args(h, Xs, Zs, M, acq, fn, score, mu, sigma, linf, &a);
  // K* in pair order, box by box: per CTA np / 8 dense boxes of one k group (32 pairs x 8 k x 2 rows), so the map
  // is [grid * np / 8 * 32 rows][16 doubles] and every box, stored or loaded, is 4 KB of consecutive bytes
  VZ_TRY(make_map(&a.mapA, a.scratch, (uint64_t)grid * (kTM / 2) * (h->np / 8), 16, 16, kTM / 2));
  static_assert(4 * kABox == kTM * kBK, "four A boxes hold one slab of K*");
  VZ_TRY(make_map(&a.mapB, a.Linv, (uint64_t)h->np, (uint64_t)h->np, (uint64_t)h->np, kBPieceRows));
  a.nsplit = nsplit;
  if (nsplit > 1) {
    VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)(nsplit + 2) * a.mpad));
    a.part = h->Tws.as<double>();
  }
  void* kargs[] = {&a};
  VZ_CUDA(cudaLaunchKernelExC(&cfg, kfn, kargs));
  VZ_CHECK_LAUNCH();
  h->launches++;
  if (nsplit > 1) {
    if (a.acq.main.kind == VZGP_ACQ_MES) k_score_finalize<true><<<(M + 255) / 256, 256, 0, h->stream>>>(a);
    else k_score_finalize<false><<<(M + 255) / 256, 256, 0, h->stream>>>(a);
    VZ_CHECK_LAUNCH();
    h->launches++;
  }
  return 0;
}

// ---------------------------------------------------------------------------
// The member loop of the multi-model launchers (ensembles, stacks, GP-UCB-PE): groups[g][e] (g < n_groups, e < per)
// is scored by launch_score on its own route, mean and stddev, into owner->pe_tmp, which launch_score does not
// touch: [2 n_groups per + 2][M] = per group mu | sd (per rows each), then linf | dummy.  Every member asks for
// `req`; member `dist` of the last group asks for `req_dist` and, when want_linf, writes the trust-region distance
// to *linf (the linf plane when *linf is null).  *planes = the first plane.  Asynchronous, capturable.
// ---------------------------------------------------------------------------
static int score_members(vzgp_handle* owner, vzgp_handle* const* const* groups, int n_groups, int per,
                         const double* Xs, const int32_t* Zs, int M, const vzgp_acq& req, int dist,
                         const vzgp_acq& req_dist, bool want_linf, double** planes, double** linf) {
  const size_t n = (size_t)n_groups * per;
  VZ_TRY(owner->pe_tmp.reserve(sizeof(double) * (2 * n + 2) * (size_t)M));
  double* t = owner->pe_tmp.as<double>();
  if (*linf == nullptr) *linf = t + 2 * n * M;
  double* dummy = t + (2 * n + 1) * M;
  for (int g = 0; g < n_groups; ++g)
    for (int e = 0; e < per; ++e) {
      const bool d = g == n_groups - 1 && e == dist;
      double* mu = t + (2 * (size_t)g * per + e) * M;
      VZ_TRY(launch_score(groups[g][e], Xs, Zs, M, d ? &req_dist : &req, dummy, mu, mu + (size_t)per * M,
                          d && want_linf ? *linf : nullptr));
    }
  *planes = t;
  return 0;
}

// ---------------------------------------------------------------------------
// GP-UCB-PE acquisition from the pieces of two models (gp_ucb_pe.py:344-381, :434-492, :221-242).
// ---------------------------------------------------------------------------
struct PeCombine {
  int mode;
  double ucb, explore, penalty, threshold;
  TrustRegion tr;
};

// ---------------------------------------------------------------------------
// Stacked residual GPs of transfer learning (StackedResidualGP, gp/gp_models.py:91-140; combine_predictions_with_aux,
// gp/transfer_learning.py:62-152): level 0 is the first prior study's GP, every further level is trained on the
// residuals of the stack below it, the last level on the current study.  Every level is a uniform ensemble of E
// members (VizierGPBandit(ensemble_size=E).set_priors trains each level with the designer's spec,
// gp_bandit.py:402-447; E = 1 is a single GP).  Per candidate, each level's prediction is the two-pass mixture of its
// members (pe_mixture: with E = 1 exactly the member's mean and stddev), then mean = sum of the level means and the
// stddevs are combined bottom-up by weighted geometric means  s <- sd_l^alpha_l * s^(1 - alpha_l)  (alpha_l from the
// degrees of freedom of the two levels, computed by the caller).  The acquisition and the non-strict trust region
// (distances to the TOP level's trials) follow.  mu_e / sd_e: [L][E][M], level-major like the handles.
// ---------------------------------------------------------------------------
struct StackEnsCombine {
  int L, E;
  double alpha[kMaxStackLevels];
  AcqFn acq;
  TrustRegion tr;
};
__global__ void __launch_bounds__(256) k_stack_ensemble_combine(int M, StackEnsCombine p,
                                                                const double* __restrict__ mu_e,
                                                                const double* __restrict__ sd_e,
                                                                const double* __restrict__ linf,
                                                                double* __restrict__ score, double* __restrict__ mu,
                                                                double* __restrict__ sigma) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const size_t level = (size_t)p.E * M;
  double mean, sd;
  pe_mixture(p.E, mu_e, sd_e, (size_t)M, m, mean, sd);
  for (int l = 1; l < p.L; ++l) {
    double mean_l, sd_l;
    pe_mixture(p.E, mu_e + l * level, sd_e + l * level, (size_t)M, m, mean_l, sd_l);
    mean += mean_l;
    sd = pow(sd_l, p.alpha[l]) * pow(sd, 1.0 - p.alpha[l]);
  }
  score[m] = tr_apply(p.tr, acq_value<false>(p.acq, mean, sd), linf[m]);
  if (mu) mu[m] = mean;
  if (sigma) sigma[m] = sd;
}

// hs[l * E + e] = member e of level l, all L E members one group of score_members in the top handle's pe_tmp;
// top-level member 0 gives the trust-region distance (the members of a level share its trials).
int launch_score_stack_ensemble(vzgp_handle* const* hs, int L, int E, const double* alphas, const double* Xs,
                                const int32_t* Zs, int M, const vzgp_acq* acq, double* score, double* mu, double* sigma,
                                double* linf, const AcqFn* fn) {
  if (M <= 0) return 0;
  const int n = L * E;
  vzgp_handle* top = hs[(L - 1) * E];
  StackEnsCombine p;
  p.L = L; p.E = E; p.acq = acq_fn_of(acq, fn);
  p.tr = trust_region_of(top, *acq, acq->tr_strict);
  const vzgp_acq req = posterior_request(acq->tr_dim_mask, acq->tr_rows);
  double *t, *linf_buf = linf;
  VZ_TRY(score_members(top, &hs, 1, n, Xs, Zs, M, req, (L - 1) * E, req, tr_needs_distance(p.tr) || linf != nullptr,
                       &t, &linf_buf));
  for (int l = 0; l < kMaxStackLevels; ++l) p.alpha[l] = l < L ? alphas[l] : 0.0;
  k_stack_ensemble_combine<<<(M + 255) / 256, 256, 0, top->stream>>>(M, p, t, t + (size_t)n * M, linf_buf, score, mu,
                                                                     sigma);
  VZ_CHECK_LAUNCH();
  top->launches++;
  return 0;
}

// ---------------------------------------------------------------------------
// Set-PE acquisition (SetPEScoreFunction, gp_ucb_pe.py:510-594): per set of q points
//   logdet(joint predictive covariance under model B)  +  penalty * sum_i min(mean_A + explore * stddev_A - threshold, 0)
//   [+ sum_i tr_set_term(dist_i) when radius <= 0.5                        _apply_trust_region_to_set, :245-269]
// One warp per set: the q x q block of the [M x M] covariance is factored in shared memory (q <= 16); a pivot that is
// not positive gives -inf like the reference's NaN -> -inf rule (:495-507).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32) k_set_pe_combine(int n_sets, int q, PeCombine p, const double* __restrict__ cov, int ldc,
                                                       const double* __restrict__ mu_a, const double* __restrict__ sd_a,
                                                       const double* __restrict__ linf, double* __restrict__ score,
                                                       double* __restrict__ sd_all) {
  __shared__ double c[16][17];
  const int s = blockIdx.x, lane = threadIdx.x;
  if (s >= n_sets) return;
  const int r0 = s * q;
  for (int e = lane; e < q * q; e += 32) c[e / q][e % q] = cov[(size_t)(r0 + e / q) * ldc + r0 + e % q];
  __syncwarp();
  if (sd_all && lane < q) sd_all[r0 + lane] = sqrt(fmax(c[lane][lane], 0.0));
  double logdet = 0.0;
  bool bad = false;
  for (int k = 0; k < q; ++k) {
    const double d = c[k][k];
    if (!(d > 0.0) || !isfinite(d)) { bad = true; break; }
    logdet += log(d);
    __syncwarp();
    const double inv = 1.0 / d;
    // right-looking LDL^T step on the trailing block: lane = row i > k
    for (int i = k + 1 + lane; i < q; i += 32) {
      const double lik = c[i][k] * inv;
      for (int j = k + 1; j <= i; ++j) c[i][j] -= lik * c[j][k];
    }
    __syncwarp();
    // keep the block symmetric for the next pivot column reads (c[j][k] with j > k is the lower part: already there)
  }
  double pen = 0.0, tr = 0.0;
  for (int i = lane; i < q; i += 32) {
    pen += fmin(mu_a[r0 + i] + p.explore * sd_a[r0 + i] - p.threshold, 0.0);
    if (p.tr.apply) tr += tr_set_term(p.tr, linf[r0 + i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    pen += __shfl_xor_sync(0xffffffffu, pen, o);
    tr += __shfl_xor_sync(0xffffffffu, tr, o);
  }
  if (lane == 0) score[s] = (bad ? -INFINITY : logdet) + p.penalty * pen + tr;
}

int launch_set_pe_combine(vzgp_handle* h, int n_sets, int q, const vzgp_pe_params* pe, const double* cov, int ldc,
                          const double* mu_a, const double* sd_a, const double* linf, double* score, double* sd_all) {
  PeCombine p;
  p.mode = 1; p.ucb = pe->ucb_coefficient; p.explore = pe->explore_coefficient;
  p.penalty = pe->penalty_coefficient; p.threshold = pe->threshold;
  p.tr = trust_region_of(h, *pe, true);
  p.tr.apply = linf != nullptr && tr_needs_distance(p.tr);
  k_set_pe_combine<<<n_sets, 32, 0, h->stream>>>(n_sets, q, p, cov, ldc, mu_a, sd_a, linf, score, sd_all);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// ---------------------------------------------------------------------------
// Uniform ensemble of E models (UniformEnsemblePredictive, stochastic_process_model.py:846-868:
// equal-weight MixtureSameFamily): mean = avg mu_e, var = avg(sd_e^2 + mu_e^2) - mean^2.
// ---------------------------------------------------------------------------
struct EnsCombine {
  int E;
  AcqFn acq;
  TrustRegion tr;
};
__global__ void k_ensemble_combine(int M, EnsCombine p, const double* __restrict__ mu_e, const double* __restrict__ sd_e,
                                   const double* __restrict__ linf, double* __restrict__ score,
                                   double* __restrict__ mu, double* __restrict__ sigma, int* __restrict__ clamp_count) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double s1 = 0.0, s2 = 0.0;
  for (int e = 0; e < p.E; ++e) {
    const double a = mu_e[(size_t)e * M + m], b = sd_e[(size_t)e * M + m];
    s1 += a;
    s2 += fma(b, b, a * a);
  }
  const double mean = s1 / p.E;
  double var = s2 / p.E - mean * mean;
  if (var < 0.0) { var = 0.0; atomicAdd(clamp_count, 1); }
  const double sd = sqrt(var);
  score[m] = tr_apply(p.tr, acq_value<false>(p.acq, mean, sd), linf[m]);
  if (mu) mu[m] = mean;
  if (sigma) sigma[m] = sd;
}

int launch_score_ensemble(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int M,
                          const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf, const AcqFn* fn) {
  if (M <= 0) return 0;
  vzgp_handle* h0 = hs[0];
  EnsCombine p;
  p.E = E; p.acq = acq_fn_of(acq, fn);
  p.tr = trust_region_of(h0, *acq, acq->tr_strict);
  const vzgp_acq req = posterior_request(acq->tr_dim_mask, acq->tr_rows);
  double *t, *linf_buf = linf;
  // all members share the trials: member 0 gives the distance
  VZ_TRY(score_members(h0, &hs, 1, E, Xs, Zs, M, req, 0, req, tr_needs_distance(p.tr) || linf != nullptr, &t, &linf_buf));
  k_ensemble_combine<<<(M + 255) / 256, 256, 0, h0->stream>>>(M, p, t, t + (size_t)E * M, linf_buf, score, mu, sigma,
                                                              h0->small.as<int>());
  VZ_CHECK_LAUNCH();
  h0->launches++;
  return 0;
}

// ---------------------------------------------------------------------------
// GP-UCB-PE over uniform ensembles (pe_ensemble.cuh): per candidate the mixtures of the E members of A and of B,
// then the UCB / PE acquisition and the strict trust region.  Outputs: score, optional mixture mean / stddev of A
// and stddev of B.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pe_ensemble_combine(int M, PeEnsCombine p, const double* __restrict__ mu_a,
                                                             const double* __restrict__ sd_a,
                                                             const double* __restrict__ mu_b,
                                                             const double* __restrict__ sd_b,
                                                             const double* __restrict__ linf, double* __restrict__ score,
                                                             double* __restrict__ mu, double* __restrict__ sigma,
                                                             double* __restrict__ sigma_all) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double mean_a, s_a, mean_b, s_b;
  pe_mixture(p.E, mu_a, sd_a, (size_t)M, m, mean_a, s_a);
  pe_mixture(p.E, mu_b, sd_b, (size_t)M, m, mean_b, s_b);
  score[m] = pe_ensemble_score(p, mean_a, s_a, s_b, linf[m]);
  if (mu) mu[m] = mean_a;
  if (sigma) sigma[m] = s_a;
  if (sigma_all) sigma_all[m] = s_b;
}

// The A members, then the B members, as the two groups of score_members in hAs[0]->pe_tmp: [4E + 2][M] =
// mu_a | sd_a | mu_b | sd_b (E rows each) | linf | dummy.  B member 0 gives the trust-region distance (all B members
// share the trials).  E = 1 is the GP-UCB-PE of two single models (vzgp_score_pe).
int launch_score_pe_ensemble(vzgp_handle* const* hAs, vzgp_handle* const* hBs, int E, const double* Xs,
                             const int32_t* Zs, int M, const vzgp_pe_params* pe, double* score, double* mu,
                             double* sigma, double* sigma_all) {
  if (M <= 0) return 0;
  vzgp_handle* h0 = hAs[0];
  const PeEnsCombine p = pe_ensemble_args(hBs[0], E, pe);
  const vzgp_acq none = posterior_request(), accb = posterior_request(pe->tr_dim_mask, pe->tr_rows);
  vzgp_handle* const* const groups[2] = {hAs, hBs};
  double *t, *linf_b = nullptr;
  VZ_TRY(score_members(h0, groups, 2, E, Xs, Zs, M, none, 0, accb, tr_needs_distance(p.tr), &t, &linf_b));
  const size_t em = (size_t)E * M;
  k_pe_ensemble_combine<<<(M + 255) / 256, 256, 0, h0->stream>>>(M, p, t, t + em, t + 2 * em, t + 3 * em, linf_b, score,
                                                                 mu, sigma, sigma_all);
  VZ_CHECK_LAUNCH();
  h0->launches++;
  return 0;
}

// ---------------------------------------------------------------------------
// Philox candidate pool: X[m, d] = U(seed, STREAM_RANDOM_POOL, 0, (index_base+m)*dc + d)
// ---------------------------------------------------------------------------
__global__ void k_random_pool(double* __restrict__ X, int64_t total, int64_t elem_base,
                              uint64_t seed, uint32_t stream, uint32_t iteration) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; e < total; e += stride)
    X[e] = philox_uniform(seed, stream, iteration, (uint64_t)(elem_base + e));
}

int launch_random_fill(vzgp_handle* h, double* X, int64_t total, int64_t elem_base, uint64_t seed,
                       uint32_t stream, uint32_t iteration) {
  if (total <= 0) return 0;
  int64_t blocks = (total + 255) / 256;
  if (blocks > (int64_t)h->sm_count * 16) blocks = (int64_t)h->sm_count * 16;
  k_random_pool<<<(unsigned)blocks, 256, 0, h->stream>>>(X, total, elem_base, seed, stream, iteration);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// ---------------------------------------------------------------------------
// Top-k by repeated arg-max (count is small: the number of suggestions).  Ordering: larger
// score first, ties -> lower index, NaN -> -inf.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool better(double v, long long i, double bv, long long bi) {
  return (v > bv) || (v == bv && i < bi);
}

// partial[b] = best of this block's slice, ignoring indices already in taken[0..ntaken)
__global__ void k_argmax_partial(const double* __restrict__ s, int64_t M,
                                 const long long* __restrict__ taken, int ntaken,
                                 ArgMax* __restrict__ partial) {
  __shared__ double sv[256];
  __shared__ long long si[256];
  double bv = -INFINITY;
  long long bi = LLONG_MAX;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < M;
       e += (int64_t)gridDim.x * blockDim.x) {
    double v = s[e];
    if (isnan(v)) v = -INFINITY;
    bool skip = false;
    for (int t = 0; t < ntaken; ++t) skip |= (taken[t] == e);
    if (!skip && better(v, e, bv, bi)) { bv = v; bi = e; }
  }
  sv[threadIdx.x] = bv;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o && better(sv[threadIdx.x + o], si[threadIdx.x + o], sv[threadIdx.x], si[threadIdx.x])) {
      sv[threadIdx.x] = sv[threadIdx.x + o];
      si[threadIdx.x] = si[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { partial[blockIdx.x].v = sv[0]; partial[blockIdx.x].i = si[0]; }
}

__global__ void k_argmax_final(const ArgMax* __restrict__ partial, int nb, long long* __restrict__ taken,
                               double* __restrict__ vals, int slot) {
  __shared__ double sv[256];
  __shared__ long long si[256];
  double bv = -INFINITY;
  long long bi = LLONG_MAX;
  for (int e = threadIdx.x; e < nb; e += blockDim.x)
    if (better(partial[e].v, partial[e].i, bv, bi)) { bv = partial[e].v; bi = partial[e].i; }
  sv[threadIdx.x] = bv;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o && better(sv[threadIdx.x + o], si[threadIdx.x + o], sv[threadIdx.x], si[threadIdx.x])) {
      sv[threadIdx.x] = sv[threadIdx.x + o];
      si[threadIdx.x] = si[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { taken[slot] = si[0]; vals[slot] = sv[0]; }
}

// Device-side top-k: results land in d_idx[count], d_val[count] (device).
int launch_topk_device(vzgp_handle* h, const double* score, int64_t M, int count, long long* d_idx,
                       double* d_val, ArgMax* d_partial, int nblocks) {
  for (int c = 0; c < count; ++c) {
    k_argmax_partial<<<nblocks, 256, 0, h->stream>>>(score, M, d_idx, c, d_partial);
    VZ_CHECK_LAUNCH();
    k_argmax_final<<<1, 256, 0, h->stream>>>(d_partial, nblocks, d_idx, d_val, c);
    VZ_CHECK_LAUNCH();
    h->launches += 2;
  }
  return 0;
}

// Gather rows: out[c, :] = X[idx[c], :]  (idx may be LLONG_MAX when fewer than count exist)
__global__ void k_gather_rows(const double* __restrict__ X, int dc, const long long* __restrict__ idx,
                              int count, int64_t M, double* __restrict__ out) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count * dc) return;
  int c = e / dc, d = e % dc;
  long long i = idx[c];
  out[e] = (i >= 0 && i < M) ? X[(size_t)i * dc + d] : 0.0;
}

int launch_gather_rows(vzgp_handle* h, const double* X, int dc, const long long* idx, int count,
                       int64_t M, double* out) {
  k_gather_rows<<<(count * dc + 255) / 256, 256, 0, h->stream>>>(X, dc, idx, count, M, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// Pack the local winners as rows [score, global index, Dc features] (fp64; indices < 2^53 exact).
__global__ void k_pack_topk(const double* __restrict__ X, int dc, const long long* __restrict__ idx,
                            const double* __restrict__ val, int count, int64_t M, int64_t index_base,
                            double* __restrict__ payload) {
  const int w = dc + 2;
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count * w) return;
  const int c = e / w, d = e % w;
  const long long i = idx[c];
  const bool ok = (i >= 0 && i < M);
  double v;
  if (d == 0) v = ok ? val[c] : -INFINITY;
  else if (d == 1) v = ok ? (double)(index_base + i) : -1.0;
  else v = ok ? X[(size_t)i * dc + (d - 2)] : 0.0;
  payload[e] = v;
}

int launch_pack_topk(vzgp_handle* h, const double* X, int dc, const long long* idx, const double* val,
                     int count, int64_t M, int64_t index_base, double* payload) {
  const int n = count * (dc + 2);
  k_pack_topk<<<(n + 255) / 256, 256, 0, h->stream>>>(X, dc, idx, val, count, M, index_base, payload);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

// Merge gathered winner rows: merge_topk_block (topk_merge.cuh), one CTA.
__global__ void __launch_bounds__(256) k_merge_topk(const double* __restrict__ rows, int n_rows, int width,
                                                    int count, double* __restrict__ out) {
  merge_topk_block<false>(rows, n_rows, width, count, out);
}

int launch_merge_topk(vzgp_handle* h, const double* rows, int n_rows, int width, int count, double* out) {
  k_merge_topk<<<1, 256, 0, h->stream>>>(rows, n_rows, width, count, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}


}  // namespace vzgp

#ifdef VZ_SCORE_TIMING
// Instrumented build only: the k_score counters (slots listed at g_score_t).  reset != 0 clears them.
extern "C" int vzgp_debug_score_timing(unsigned long long* out, int reset) {
  if (cudaMemcpyFromSymbol(out, vzgp::g_score_t, sizeof(vzgp::g_score_t)) != cudaSuccess) return -2;
  if (reset) {
    unsigned long long z[vzgp::kScoreCounters] = {};
    if (cudaMemcpyToSymbol(vzgp::g_score_t, z, sizeof(z)) != cudaSuccess) return -2;
  }
  return 0;
}
#endif
