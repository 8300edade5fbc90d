// The W = K* . Linv^T contraction of the scoring path on the Hopper tensor cores (wgmma, s8 x s8 -> s32),
// by an Ozaki-style exact integer split of the fp64 operands.
//
// Same contract as k_score (score.cu): posterior mean / variance + UCB + trust region for a candidate pool;
// replaces BayesianScoringFunction.score_with_aux (acquisitions.py:177-207).  The tensor cores have no fp64 kind
// beyond DMMA; wgmma multiplies 8-bit integers with exact 32-bit accumulation.  So both operands are written as
// fixed-point numbers of 7 base-256 digits relative to a power-of-two row scale, with BALANCED digits,
//     K*[i,k]   = 2^ea   * sum_{s=1..7} a_s[i,k] 2^(-8s)      a_s in [-128,127]
//     Linv[j,k] = 2^eb_j * sum_{t=1..7} b_t[j,k] 2^(-8t)      b_t in [-128,127]
// i.e. 55 bits below the row maximum - what fp64 carries for the entries that dominate the sum - and
//     W[i,j] = 2^(ea+eb_j) * sum_{g=2..8} 2^(-8g) G_g[i,j],   G_g = sum_{s+t=g} a_s b_t^T   (28 digit products)
// where every G_g is an EXACT int32 (|G_g| <= 7 * np * 128 * 128 < 2^31 for np <= 4096, the limit of this path).
// Products with s + t > 8 are dropped.  With balanced digits they have zero mean and sum to ~1e-15 of the
// row-scale product (unsigned digits would add a one-sided 3e-13: measured in tools/ozaki_emulation.py), the
// same order as the rounding of an fp64 accumulation.
//
// One persistent CTA per SM, 64 candidates per tile:
//   phase 1   (8 K* warps)  K* tile by 64-column steps as in k_score; mu and the L-inf distance on the fly;
//             every K* value is cut into its 7 digits and stored to a CTA-private scratch
//             [7 digit planes][64 candidates][np] (L2 resident).
//   phase 2   (one consumer warpgroup)  D[64 x 32] (s32 registers) += A B^T, A = a Linv digit plane (j tile of
//             64 rows), B = a K* digit plane of 32 candidates; 7 accumulator groups (g).  Per 128-byte k chunk the
//             14 planes are TMA-loaded into one of two stages, one chunk ahead of its 112 wgmma.
//   epilogue  (the same warpgroup) recombine the 7 groups in 64-bit integers, scale, square and add into
//             per-candidate sums; after the last j tile: variance, sigma, UCB, trust region.
#include <cuda.h>

#include <climits>
#include <cstring>

#include "launchers.h"
#include "score_small.cuh"
#include "tiles.cuh"

#ifdef VZ_I8_TIMING
namespace vzgp { __device__ long long g_i8_t[16]; }
#define VZ_I8T_DECL long long t_a = 0, t_b = 0; (void)t_a; (void)t_b
#define VZ_I8T_START(v) do { v = clock64(); } while (0)
#define VZ_I8T_ADD(slot, v) do { if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) g_i8_t[slot] += clock64() - (v); } while (0)
#else
#define VZ_I8T_DECL do {} while (0)
#define VZ_I8T_START(v) do {} while (0)
#define VZ_I8T_ADD(slot, v) do {} while (0)
#endif

namespace vzgp {

namespace {

// The consumer warpgroup needs 160 registers per thread (112 accumulators); ptxas gives all threads that budget.
constexpr int kKWarps = 8;                    // K* warps (phase 1)
constexpr int kEWarps = 4;                    // the consumer warpgroup: MMA issue and epilogue
constexpr int kI8Threads = (kKWarps + kEWarps) * 32;
constexpr int kDigits = 7;
constexpr int kGroups = 7;                    // g = s + t - 2 in [0, 6]
constexpr int kJT = 64;                       // Linv rows per j tile = wgmma M
constexpr int kCN = 32;                       // candidates per wgmma = N (half of the 64-candidate tile)
constexpr int kKC = 128;                      // bytes (= k values) per chunk: one 128-byte swizzle atom per row
constexpr int kAPlaneBytes = kJT * kKC;       // 8 KB: one digit plane of a j tile x k chunk
constexpr int kBPlaneBytes = kCN * kKC;       // 4 KB: one digit plane of a candidate half x k chunk
constexpr int kStageBytes = kDigits * (kAPlaneBytes + kBPlaneBytes);   // 84 KB
constexpr int kRingBytes = 2 * kStageBytes;   // 168 KB

struct I8Args {
  alignas(64) CUtensorMap mapK;   // K* digit scratch as u8 [grid*7*64 rows][np], box 32 x 128, SWIZZLE_128B
  alignas(64) CUtensorMap mapL;   // Linv digit planes as u8 [7][np][np], box 1 x 64 x 128, SWIZZLE_128B
  ScoreArgs s;                    // candidates, model, outputs (mapA / mapB / scratch unused)
  uint8_t* kdig;                  // [grid][nbuf][7][64][np]
  int nbuf;                       // 2: phase 1 of the next tile overlaps phase 2; 1: back to back (large Dc)
  int misc_bytes;                 // shared memory between the operand ring and the (nbuf = 2) phase-1 staging
  int sb_bufs;                    // trial staging buffers of phase 1: 2 (copy of step jb + 1 under the math of jb) or 1
  const double* lscale;           // [np]  2^(ea + eb_j - 32)
  double kscale;                  // 2^(56 - ea)
};

// mbarrier wait that turns a protocol error into a trap (cudaErrorLaunchFailure) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, unsigned parity) {
  unsigned ok, spins = 0;
  unsigned long long t0 = 0;
  for (;;) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (ok) return;
    if ((++spins & 0xfffu) == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t0 == 0) t0 = t;
      else if (t - t0 > 20000000000ull) __trap();   // 20 s: far beyond any wait of a healthy run, time-sliced GPUs included
    }
  }
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major operand tile in the 128-byte-swizzle layout TMA writes: rows
// of 128 bytes, 8-row groups 1024 bytes apart (stride byte offset), swizzle mode 1 (128B) in bits 62-63.  The tile
// base is 1024-byte aligned; a 32-byte k step inside the atom adds 2 to the (16-byte unit) start address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// D[64 x 32] (+)= A[64 x 32] B[32 x 32]^T, s8 operands from shared memory, s32 accumulators in registers.
__device__ __forceinline__ void wgmma_i8(int32_t (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads or writes across a wgmma fence / wait.
__device__ __forceinline__ void acc_fence(int32_t (&acc)[kGroups][16]) {
#pragma unroll
  for (int g = 0; g < kGroups; ++g)
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(acc[g][i])::"memory");
}
// Power-of-two scale exponent e with |x| 2^-e <= 0.498 for |x| <= m: the top balanced digit stays in [-128, 127].
__host__ __device__ inline int balanced_scale_exp(double m) {
  int e = 0;
  const double f = frexp(m, &e);
  return f < 0.996 ? e + 1 : e + 2;
}
__device__ __forceinline__ void st_u16_keep(void* p, uint16_t v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.u16 [%0], %1, %2;\n" ::"l"(p), "h"(v), "l"(policy) : "memory");
}

__device__ __forceinline__ void g_i8_t_tiles() {
#ifdef VZ_I8_TIMING
  g_i8_t[15] += 1;
#endif
}

// Hand-over between the K* warps and the consumer warpgroup by mbarriers only:
//   kready[b]  K* warps -> consumer: digit planes / mu / L-inf of the tile in buffer b are complete
//   kfree[b]   consumer -> K* warps: the tile that used buffer b is finished (all its TMA reads are consumed)
//   full[s]    TMA -> consumer: operand stage s has landed
// nbuf = 2 overlaps the phases (digit scratch and phase-1 staging have their own memory); nbuf = 1 (large Dc:
// the staging does not fit next to the operand ring) runs them back to back with the staging aliased onto the ring.
template <bool WITH_LINF, bool GENERIC>
__global__ void __launch_bounds__(kI8Threads, 1) k_score_i8(const __grid_constant__ I8Args ia) {
  const ScoreArgs& a = ia.s;
  extern __shared__ double smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(smem_raw) +
                  ((1024u - (static_cast<unsigned>(__cvta_generic_to_shared(smem_raw)) & 1023u)) & 1023u);
  constexpr int LD = kLD1;
  const int dc = a.kp.dc, dk = a.kp.dk, np = a.np, nbuf = ia.nbuf;
  uint8_t* ring = smem;                                  // [2 stages][7 A planes | 7 B planes]
  double* s_alpha = reinterpret_cast<double*>(smem + kRingBytes);   // [2][64]
  double* s_mu = s_alpha + 128;                          // [2][64]
  double* s_linf = s_mu + 128;                           // [2][64]
  double* s_red = s_linf + 128;                          // [4][64] candidate sums of the four consumer warps
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_red + 256);
  uint64_t* full = bars;                       // [2]
  uint64_t* kready = bars + 2;                 // [2]
  uint64_t* kfree = kready + 2;                // [2]
  int32_t* za = reinterpret_cast<int32_t*>(kfree + 2);   // [dk][LD]
  int32_t* zb = za + dk * LD;                            // [dk][LD]
  uint8_t* s_mask = reinterpret_cast<uint8_t*>(zb + dk * LD);  // [kMaxDc]
  // phase-1 staging: behind everything else (nbuf = 2) or aliased onto the operand ring (nbuf = 1)
  double* stage = nbuf == 2 ? reinterpret_cast<double*>(smem + ((kRingBytes + ia.misc_bytes + 15) & ~15)) : reinterpret_cast<double*>(smem);
  double* sa = stage;                                    // [dc][LD]     candidates (transposed)
  double* sb = sa + dc * LD;                             // [2][dc][LD]  trials, double buffered

  // the warp index through a shuffle: provably warp-uniform, so the role branches below are uniform branches
  const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const bool is_kwarp = warp < kKWarps;
  if (tid < kMaxDc) s_mask[tid] = a.tr.mask[tid];
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) mbar_init(full + i, 1);
    for (int i = 0; i < 2; ++i) { mbar_init(kready + i, kKWarps * 32); mbar_init(kfree + i, kEWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  const int ntiles = (a.M + kTM - 1) / kTM;
  const int njt = np / kJT;

  if (is_kwarp) {
    // ================= K* warps: phase 1 of every tile, one tile ahead of phase 2 =================
    // 256 threads, 2 x 4 outputs each on each half of the 64 x 64 block: rows 2 ty + i, columns (j/2) 32 + 2 tx + j%2
    // (ty = tid / 16 + 16 p for the row halves p, tx = tid % 16)
    struct GP {
      __device__ static int row_of(int ty, int i) { return ty * 2 + i; }
      __device__ static int col_of(int tx, int j) { return (j >> 1) * 32 + tx * 2 + (j & 1); }
    };
    constexpr int kKT = kKWarps * 32;
    constexpr int kRowSets = kTM * 16 / (2 * kKT);
    auto ksync = [&]() { asm volatile("bar.sync 1, %0;\n" ::"n"(kKT) : "memory"); };
    const int ty0 = tid / 16, tx = tid % 16;
    // the digits are written a tile ahead of their use: ask L2 to evict them last (the dead ones are discarded by the
    // epilogue warps), so that they are still resident when phase 2 streams them
    uint64_t keep_policy;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;\n" : "=l"(keep_policy));
    const double* XTs = a.XT;
    const double* XTu = a.XT + xt_plane(1, dc, np);
    unsigned it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int m0 = tile * kTM;
      const int kb = it % nbuf;
      VZ_I8T_DECL;
      VZ_I8T_START(t_a);
      mbar_wait_bounded(kfree + kb, ((it / nbuf) & 1) ^ 1);   // the tile that used this buffer is finished
      if (tid == 0) { VZ_I8T_ADD(12, t_a); }
      VZ_I8T_START(t_a);
      uint8_t* kd = ia.kdig + ((size_t)blockIdx.x * nbuf + kb) * kDigits * kTM * np;
      for (int e = tid; e < kTM * dc; e += kKT) {
        const int r = e / dc, d = e - r * dc;
        const int gr = m0 + r;
        const double v = gr < a.M ? __ldg(a.Xs + (size_t)gr * dc + d) : 0.0;
        sa[d * LD + r] = WITH_LINF ? v : v * a.kp.inv_ls_c[d];
      }
      if (dk > 0) stage_rows_T_i32(a.Zs, a.M, dk, m0, kTM, za, LD, kKT);
      auto stage_trials = [&](int jb, int buf) {
        double* dst = sb + buf * dc * LD;
        const double* src = WITH_LINF ? XTu : XTs;
        for (int c = tid; c < dc * 32; c += kKT) {       // dc rows x 32 chunks of 16 B
          const int d = c >> 5, q = c & 31;
          cp_async16(dst + d * LD + q * 2, src + (size_t)d * np + jb * 64 + q * 2, true);
        }
        if (tid < 32) cp_async16(s_alpha + buf * 64 + tid * 2, a.alpha + jb * 64 + tid * 2, true);
      };
      double mu_part[kRowSets][2], lmin[kRowSets][2];
#pragma unroll
      for (int p = 0; p < kRowSets; ++p)
#pragma unroll
        for (int i = 0; i < 2; ++i) { mu_part[p][i] = 0.0; lmin[p][i] = INFINITY; }
      const int nj = np / 64;
      const bool dbl = ia.sb_bufs == 2;
      stage_trials(0, 0);
      cp_async_commit();
      for (int jb = 0; jb < nj; ++jb) {
        const int buf = dbl ? (jb & 1) : 0;
        if (dbl) {
          if (jb + 1 < nj) stage_trials(jb + 1, buf ^ 1);
          cp_async_commit();
          cp_async_wait<1>();
        } else {                       // one staging buffer (large Dc): the copy of step jb was issued after step jb - 1
          cp_async_wait<0>();
        }
        ksync();
        if (dk > 0) {
          stage_rows_T_i32(a.Z, np, dk, jb * 64, 64, zb, LD, kKT);
          ksync();
        }
#pragma unroll
        for (int p = 0; p < kRowSets; ++p) {
          const int ty = ty0 + p * (kKT / 16);
          constexpr int zoff = 0;
          const double* sbj = sb + buf * dc * LD + zoff;
          const double* alj = s_alpha + buf * 64 + zoff;
          double d2[2][4], lf[2][4];
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { d2[i][j] = 0.0; lf[i][j] = 0.0; }
          for (int d = 0; d < dc; ++d) {
            const double2 av = *reinterpret_cast<const double2*>(sa + d * LD + GP::row_of(ty, 0));
            const double2 b0 = *reinterpret_cast<const double2*>(sbj + d * LD + GP::col_of(tx, 0));
            const double2 b1 = *reinterpret_cast<const double2*>(sbj + d * LD + GP::col_of(tx, 2));
            const double aa[2] = {av.x, av.y}, bb[4] = {b0.x, b0.y, b1.x, b1.y};
            if (WITH_LINF) {
              const double w = a.kp.inv_ls2_c[d];
              const bool in_tr = s_mask[d] != 0;
#pragma unroll
              for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const double df = aa[i] - bb[j];
                  d2[i][j] = fma(df * df, w, d2[i][j]);
                  if (in_tr) lf[i][j] = fmax(lf[i][j], fabs(df));
                }
            } else {
#pragma unroll
              for (int i = 0; i < 2; ++i)
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
            for (int i = 0; i < 2; ++i) {
              const int avz = za[k * LD + GP::row_of(ty, i)];
#pragma unroll
              for (int j = 0; j < 4; ++j) d2[i][j] += (avz != zb[k * LD + zoff + GP::col_of(tx, j)]) ? w : 0.0;
            }
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            long long q[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int cj = zoff + GP::col_of(tx, j);
              const bool valid = (jb * 64 + cj) < a.n_valid;
              const double kv = valid ? matern52(d2[i][j], a.kp.sf2) : 0.0;
              mu_part[p][i] = fma(kv, alj[GP::col_of(tx, j)], mu_part[p][i]);
              if (WITH_LINF && (jb * 64 + cj) < a.tr.rows) lmin[p][i] = fmin(lmin[p][i], lf[i][j]);
              q[j] = __double2ll_rn(kv * ia.kscale);    // |q| < 2^55
            }
            uint8_t* row = kd + (size_t)GP::row_of(ty, i) * np + jb * 64 + zoff;
            // balanced base-256 digits, least significant first: digit = low byte (two's complement), carry (q + 128) >> 8
#pragma unroll
            for (int s = kDigits - 1; s >= 0; --s) {
              uint8_t* p = row + (size_t)s * kTM * np;
              st_u16_keep(p + GP::col_of(tx, 0), (uint16_t)((q[0] & 255ll) | ((q[1] & 255ll) << 8)), keep_policy);
              st_u16_keep(p + GP::col_of(tx, 2), (uint16_t)((q[2] & 255ll) | ((q[3] & 255ll) << 8)), keep_policy);
#pragma unroll
              for (int j = 0; j < 4; ++j) q[j] = (q[j] + 128) >> 8;
            }
          }
        }
        ksync();
        if (!dbl && jb + 1 < nj) {     // everybody is done with the buffer: refill it (latency exposed, large Dc only)
          stage_trials(jb + 1, 0);
          cp_async_commit();
        }
      }
      cp_async_wait<0>();
#pragma unroll
      for (int p = 0; p < kRowSets; ++p)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) {
            mu_part[p][i] += __shfl_xor_sync(0xffffffffu, mu_part[p][i], o);
            if (WITH_LINF) lmin[p][i] = fmin(lmin[p][i], __shfl_xor_sync(0xffffffffu, lmin[p][i], o));
          }
          if (tx == 0) {
            s_mu[kb * 64 + GP::row_of(ty0 + p * (kKT / 16), i)] = mu_part[p][i];
            s_linf[kb * 64 + GP::row_of(ty0 + p * (kKT / 16), i)] = lmin[p][i];
          }
        }
      fence_proxy_async();  // generic-proxy writes (digit scratch, aliased smem) before async-proxy (TMA) accesses
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(kready + kb)) : "memory");
      if (tid == 0) { VZ_I8T_ADD(0, t_a); }
    }
  } else {
    // ================= consumer warpgroup: operand loads, wgmma, epilogue =================
    constexpr int kET = kEWarps * 32;
    auto esync = [&]() { asm volatile("bar.sync 2, %0;\n" ::"n"(kET) : "memory"); };
    const int etid = tid - kKWarps * 32;
    const int ew = etid >> 5;                    // consumer warp: rows 16 ew .. 16 ew + 15 of the j tile
    int clamped = 0;
    unsigned it = 0;
    unsigned n_ld = 0, n_use = 0;                // chunks loaded / consumed: stage n & 1, phase parity (n >> 1) & 1
    const bool can_discard = (np % kKC) == 0;    // discard.L2 wants 128-byte aligned lines
    int32_t acc[kGroups][16];
#pragma unroll
    for (int g = 0; g < kGroups; ++g)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[g][i] = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int m0 = tile * kTM;
      const int kb = it % nbuf;
      const int krow0 = ((int)blockIdx.x * nbuf + kb) * kDigits * kTM;
      const uint8_t* kdt = ia.kdig + (size_t)krow0 * np;
      VZ_I8T_DECL;
      VZ_I8T_START(t_a);
      // Each candidate sum s_red[ew][c] is owned by one lane (c = 32 half + 8 q + 2 lane + cc, lane < 4).
      if (lane < 4) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            s_red[ew * 64 + h * kCN + 8 * q + 2 * lane] = 0.0;
            s_red[ew * 64 + h * kCN + 8 * q + 2 * lane + 1] = 0.0;
          }
      }
      mbar_wait_bounded(kready + kb, (it / nbuf) & 1);     // the tile's digit planes, mu and L-inf are complete
      auto load = [&](int jt, int half, int kc) {
        if (etid == 0) {
          const int st = n_ld & 1;
          uint8_t* dst = ring + st * kStageBytes;
          mbar_expect_tx(full + st, kStageBytes);
          for (int t = 0; t < kDigits; ++t) tma_load_3d(dst + t * kAPlaneBytes, &ia.mapL, kc * kKC, jt * kJT, t, full + st);
          for (int s = 0; s < kDigits; ++s)
            tma_load_2d(dst + kDigits * kAPlaneBytes + s * kBPlaneBytes, &ia.mapK, kc * kKC, krow0 + s * kTM + half * kCN, full + st);
        }
        __syncwarp();
        ++n_ld;
      };
      // The chunks of the tile in order: j tiles descending (k chunk kc is last needed by j tile 2 kc, so the digit
      // scratch dies front to back), the two candidate halves, k chunks 0 .. jt / 2 (Linv is lower triangular).
      int jt = njt - 1, half = 0, kc = 0;
      load(jt, half, kc);
      for (;;) {
        int jt_next = jt, half_next = half, kc_next = kc + 1;
        if (kc_next > (jt >> 1)) {
          kc_next = 0;
          if (++half_next == 2) { half_next = 0; --jt_next; }
        }
        const bool block_done = kc_next == 0;      // the accumulators of (jt, half) are complete after this chunk
        const bool more = jt_next >= 0;
        const int st = n_use & 1;
        mbar_wait_bounded(full + st, (n_use >> 1) & 1);
        ++n_use;
        const int ksteps = min(4, (jt * kJT + kJT - kc * kKC) / 32);   // k beyond the j tile's last row is zero
        const uint32_t abase = smem_u32(ring + st * kStageBytes), bbase = abase + kDigits * kAPlaneBytes;
        if (kc == 0) {                             // the epilogue of the previous block has read the accumulators
          acc_fence(acc);
          wgmma_fence();
        }
#pragma unroll
        for (int t = 0; t < kDigits; ++t) {
          const uint64_t da = wgmma_desc_sw128(abase + t * kAPlaneBytes);
#pragma unroll
          for (int s = 0; s + t < kGroups; ++s) {     // digit pair (s+1, t+1): group g = s + t
            const uint64_t db = wgmma_desc_sw128(bbase + s * kBPlaneBytes);
            for (int kk = 0; kk < ksteps; ++kk)
              wgmma_i8(acc[s + t], da + 2 * kk, db + 2 * kk, (kc > 0 || kk > 0 || t > 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                           // the previous chunk's wgmma are done: its stage can be refilled
        if (more) load(jt_next, half_next, kc_next);
        if (block_done) {
          wgmma_wait<0>();
          acc_fence(acc);
          // accumulator i of this thread: Linv row 16 ew + lane / 4 + 8 ((i >> 1) & 1), candidate 8 (i >> 2) + 2 (lane % 4) + (i & 1)
          const int j0 = jt * kJT + ew * 16 + (lane >> 2);
          const double sc[2] = {__ldg(ia.lscale + j0), __ldg(ia.lscale + j0 + 8)};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            double v[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              v[c] = 0.0;
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                const int i = 4 * q + 2 * r + c;
                // sum_g G_g 2^(-8(g+2)) = 2^-32 (hi + lo 2^-32),  hi = G0 2^16 + G1 2^8 + G2,  lo = G3 2^24 + ... + G6
                const long long hi = ((long long)acc[0][i] << 16) + ((long long)acc[1][i] << 8) + (long long)acc[2][i];
                const long long lo = ((long long)acc[3][i] << 24) + ((long long)acc[4][i] << 16) +
                                     ((long long)acc[5][i] << 8) + (long long)acc[6][i];
                const double w = sc[r] * fma((double)lo, 0x1p-32, (double)hi);
                v[c] += w * w;
              }
              // sum over the 8 row lanes (fixed order)
#pragma unroll
              for (int o = 4; o < 32; o <<= 1) v[c] += __shfl_xor_sync(0xffffffffu, v[c], o);
            }
            if (lane < 4) {
              double* red = s_red + ew * 64 + half * kCN + 8 * q + 2 * lane;
              red[0] += v[0];
              red[1] += v[1];
            }
          }
          if (can_discard && half == 1 && (jt & 1) == 0) {
            // last use of k chunk jt / 2 of this tile's K* digits: drop its lines from L2 without a write-back
            for (int i = etid; i < kDigits * kTM; i += kET)
              asm volatile("discard.global.L2 [%0], 128;\n" ::"l"(kdt + (size_t)i * np + (size_t)(jt >> 1) * kKC) : "memory");
          }
        }
        if (!more) break;
        jt = jt_next; half = half_next; kc = kc_next;
      }
      esync();
      if (etid < kTM) {
        const int r = etid, m = m0 + r;
        if (m < a.M) {
          const double rs = (s_red[r] + s_red[64 + r]) + (s_red[128 + r] + s_red[192 + r]);
          emit_score<GENERIC>(a, m, rs, s_mu[kb * 64 + r], s_linf[kb * 64 + r], clamped);
        }
      }
      esync();             // s_red and s_mu[kb] are consumed
      if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(kfree + kb)) : "memory");
      if (etid == 0) { VZ_I8T_ADD(3, t_a); if (blockIdx.x == 0) g_i8_t_tiles(); }
    }
    if (clamped) atomicAdd(a.clamp_count, clamped);
  }
}

// Linv (lower, fp64, [np x np]) -> 7 balanced base-256 digit planes relative to the row maximum, and the
// per-row scale 2^(ea + eb_j - 32) of the recombination.  One CTA per row.
__global__ void __launch_bounds__(128) k_slice_linv(const double* __restrict__ Linv, int np, int ea,
                                                    uint8_t* __restrict__ planes, double* __restrict__ lscale) {
  const int j = blockIdx.x, tid = threadIdx.x;
  __shared__ double s_max[4];
  const double* row = Linv + (size_t)j * np;
  double m = 0.0;
  for (int k = tid; k <= j; k += 128) m = fmax(m, fabs(row[k]));
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((tid & 31) == 0) s_max[tid >> 5] = m;
  __syncthreads();
  m = fmax(fmax(s_max[0], s_max[1]), fmax(s_max[2], s_max[3]));
  const int eb = (m > 0.0 && isfinite(m)) ? balanced_scale_exp(m) : 0;
  const double sc = ldexp(1.0, 56 - eb);
  for (int k = tid; k < np; k += 128) {
    const double x = (k <= j && isfinite(m)) ? row[k] : 0.0;
    long long q = __double2ll_rn(x * sc);
#pragma unroll
    for (int t = kDigits - 1; t >= 0; --t) {
      planes[((size_t)t * np + j) * np + k] = (uint8_t)(q & 255ll);
      q = (q + 128) >> 8;
    }
  }
  if (tid == 0) lscale[j] = ldexp(1.0, ea + eb - 32);
}

// shared memory behind the operand ring: alpha, mu, L-inf, reduction, barriers, categorical rows, mask
size_t score_i8_misc_bytes(int dk) {
  return sizeof(double) * (128 + 128 + 128 + 256) + sizeof(uint64_t) * 6 + sizeof(int32_t) * dk * 2 * kLD1 + kMaxDc;
}
size_t score_i8_stage_bytes(int dc, int sb_bufs = 2) { return sizeof(double) * (1 + sb_bufs) * dc * kLD1; }
size_t score_i8_smem_bytes(int dc, int dk, int nbuf, int sb_bufs = 2) {
  return 1024 + kRingBytes + ((score_i8_misc_bytes(dk) + 15) & ~size_t(15)) +
         (nbuf == 2 ? score_i8_stage_bytes(dc, sb_bufs) : 0);
}
// Shared-memory plan: overlap the phases (nbuf = 2) whenever the phase-1 staging fits next to the operand ring, giving
// up the second trial buffer for larger Dc; otherwise back to back with the staging aliased onto the ring.
struct I8Plan { int nbuf, sb_bufs; };
I8Plan score_i8_plan(int dc, int dk) {
  for (int sb_bufs = 2; sb_bufs >= 1; --sb_bufs)
    if (score_i8_smem_bytes(dc, dk, 2, sb_bufs) <= 227 * 1024) return {2, sb_bufs};
  return {1, 2};
}

}  // namespace

bool score_i8_eligible(const vzgp_handle* h, int M) {
  if (h->kp.use_linear || h->np < kKC || h->np > 4096 || h->dc < 1) return false;
  if (score_i8_stage_bytes(h->dc) > (size_t)kRingBytes) return false;
  const int ntiles = (M + kTM - 1) / kTM;
  return ntiles >= h->sm_count;          // enough tiles for one CTA per SM (no column split on this path)
}

int launch_score_i8(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                    double* score, double* mu, double* sigma, double* linf, const AcqFn* fn) {
  const int np = h->np;
  const int ntiles = (M + kTM - 1) / kTM;
  const int grid = ntiles < h->sm_count ? ntiles : h->sm_count;
  const int ea = balanced_scale_exp(h->kp.sf2);   // K* <= sf2
  if (!h->i8_ready) {
    VZ_TRY(h->i8_planes.reserve((size_t)kDigits * np * np));
    VZ_TRY(h->i8_scale.reserve(sizeof(double) * np));
    k_slice_linv<<<np, 128, 0, h->stream>>>(h->Linv.as<double>(), np, ea, h->i8_planes.as<uint8_t>(), h->i8_scale.as<double>());
    VZ_CHECK_LAUNCH();
    h->launches++;
    h->i8_ready = true;
  }
  const I8Plan plan = score_i8_plan(h->dc, h->dk);
  const int nbuf = plan.nbuf;
  VZ_TRY(h->i8_kdig.reserve((size_t)grid * nbuf * kDigits * kTM * np));
  I8Args ia;
  memset(&ia, 0, sizeof(ia));
  ScoreArgs& a = ia.s;
  fill_score_args(h, Xs, Zs, M, acq, fn, score, mu, sigma, linf, &a);
  ia.kdig = h->i8_kdig.as<uint8_t>();
  ia.lscale = h->i8_scale.as<double>();
  ia.kscale = ldexp(1.0, 56 - ea);
  ia.nbuf = nbuf;
  ia.sb_bufs = plan.sb_bufs;
  ia.misc_bytes = (int)score_i8_misc_bytes(h->dk);
  {
    const uint64_t dims[2] = {(uint64_t)np, (uint64_t)grid * nbuf * kDigits * kTM};
    const uint64_t strides[1] = {(uint64_t)np};
    const uint32_t box[2] = {(uint32_t)kKC, (uint32_t)kCN};
    // 128-byte L2 promotion: a 256-byte one would pull the neighbouring k chunk's (already discarded) line back in
    VZ_TRY(make_tensor_map_u8(&ia.mapK, ia.kdig, 2, dims, strides, box, false));
  }
  {
    const uint64_t dims[3] = {(uint64_t)np, (uint64_t)np, (uint64_t)kDigits};
    const uint64_t strides[2] = {(uint64_t)np, (uint64_t)np * np};
    const uint32_t box[3] = {(uint32_t)kKC, (uint32_t)kJT, 1u};
    VZ_TRY(make_tensor_map_u8(&ia.mapL, h->i8_planes.as<uint8_t>(), 3, dims, strides, box));
  }
  const bool need_linf = (linf != nullptr) || tr_needs_distance(a.tr);
  const size_t sm = score_i8_smem_bytes(h->dc, h->dk, nbuf, plan.sb_bufs);
  if (sm > 227 * 1024) { set_error("k_score_i8 needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
  const bool generic = !acq_fn_is_ucb(a.acq);
  const void* kfn = generic ? (need_linf ? (const void*)k_score_i8<true, true> : (const void*)k_score_i8<false, true>)
                            : (need_linf ? (const void*)k_score_i8<true, false> : (const void*)k_score_i8<false, false>);
  VZ_TRY(raise_dyn_smem(kfn, sm));
  void* kargs[] = {&ia};
  VZ_CUDA(cudaLaunchKernel(kfn, dim3(grid), dim3(kI8Threads), kargs, sm, h->stream));
  VZ_CHECK_LAUNCH();
  h->launches++;
  h->i8_launches++;
  h->score_grid = grid;
  return 0;
}

}  // namespace vzgp

#ifdef VZ_I8_TIMING
// Debug builds only (make EXTRA=-DVZ_I8_TIMING): clock64 sums of CTA 0.  [0] phase 1, [3] whole tile (consumer),
// [12] K* warps waiting for a free digit buffer, [15] tiles.  reset != 0 clears the counters.
extern "C" int vzgp_debug_i8_timing(long long* out, int reset) {
  if (cudaMemcpyFromSymbol(out, vzgp::g_i8_t, sizeof(long long) * 16) != cudaSuccess) return -2;
  if (reset) {
    long long z[16] = {};
    if (cudaMemcpyToSymbol(vzgp::g_i8_t, z, sizeof(z)) != cudaSuccess) return -2;
  }
  return 0;
}
#endif
