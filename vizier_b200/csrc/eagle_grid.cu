// Multi-CTA persistent Eagle loop for mid-size studies (64 < N, batch <= 512 candidates).
//
// The default designers run 3000 sequential suggest -> score -> update iterations of 25 candidates
// (vectorized_base.py:431-495).  As separate launches one iteration is five kernels (suggest, K* blocks,
// W blocks, finalize, update), ~45 us at N = 1000 even when replayed from a CUDA graph, most of it launch
// and drain latency.  Here ONE cooperative launch runs the whole loop: the same device functions
// (eagle_dev.cuh, score_small.cuh) execute as phases of a persistent grid, separated by a light
// grid-wide barrier (one atomic per CTA on a monotone counter + acquire spin).  Population state and
// the K* / partial-sum workspaces stay in global memory (L2 resident).
//
//   phase S  one CTA per batch fly     eagle_suggest_cta              -> batch
//   phase C  N/64 x tiles work items   cross_small_block (per model)  -> K* scratch, partial mu / L-inf
//   phase V  N/16 x tiles work items   var_small_block  (per model)   -> partial sum W^2
//   phase U  CTA 0                     fixed-order finalize (+ GP-UCB-PE combine), eagle_update_block
//
// k_eagle_grid_pe_ensemble is the same loop for GP-UCB-PE over uniform ensembles (pe_ensemble.cuh): phases C and V
// enumerate the work items of all 2E member models, phase U finalises every member and forms the mixture score.
#include "eagle_dev.cuh"
#include "pe_ensemble.cuh"
#include "score_small.cuh"

namespace vzgp {

struct GridArgs {
  EagleDev e;
  ScoreArgs a;        // model A (UCB: the model)
  ScoreArgs b;        // model B (GP-UCB-PE only)
  int pe_mode;        // -1: UCB on a; 0 / 1: GP-UCB-PE (vzgp_pe_params.mode)
  int wl_a, wl_b;     // trust-region distance wanted from a / b
  double ucb, explore, penalty, threshold;
  TrustRegion tr;     // GP-UCB-PE: strict trust region on b's distance
  int steps;
  unsigned* barrier;  // zeroed by the host before the launch
};

__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned nblocks, unsigned& generation) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned target = (++generation) * nblocks;
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}

template <bool GENERIC>
__global__ void __launch_bounds__(kSmallThreads) k_eagle_grid(const __grid_constant__ GridArgs g) {
  extern __shared__ double smem[];
  const EagleDev& e = g.e;
  const int tid = threadIdx.x;
  const unsigned nblk = gridDim.x;
  unsigned gen = 0;
  const bool two = g.pe_mode >= 0;
  const int ntiles = (e.B + kTM - 1) / kTM;
  const int rgs = ntiles == 1 ? (e.B + 15) / 16 : 4;     // 16-candidate row groups per tile
  const int c_a = (g.a.np / 64) * ntiles * rgs, c_b = two ? (g.b.np / 64) * ntiles * rgs : 0;
  const int v_a = (g.a.np / kVarCols) * ntiles, v_b = two ? (g.b.np / kVarCols) * ntiles : 0;
#ifdef VZ_EAGLE_TIMING
  long long c_[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t0 = clock64(), t1;
#define VZ_GT(i) do { t1 = clock64(); c_[i] += t1 - t0; t0 = t1; } while (0)
#else
#define VZ_GT(i) do {} while (0)
#endif
  for (int it = 0; it < g.steps; ++it) {
    // ---- S: new batch ----
    for (int fb = blockIdx.x; fb < e.B; fb += nblk) eagle_suggest_cta<kSmallThreads>(e, fb, smem);   // one CTA per fly
    VZ_GT(0);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(1);
    // ---- C: K* blocks, partial mean / distance ----
    for (int w = blockIdx.x; w < c_a + c_b; w += nblk) {
      const bool on_b = w >= c_a;
      const ScoreArgs& s = on_b ? g.b : g.a;
      const int q = on_b ? w - c_a : w, nmb = s.np / 64;
      const int jb = q % nmb, tr = q / nmb, tile = tr / rgs, rg = tr % rgs;
      if (on_b ? g.wl_b : g.wl_a) cross_small_block<true>(s, jb, tile, rg, smem);
      else cross_small_block<false>(s, jb, tile, rg, smem);
      __syncthreads();
    }
    VZ_GT(2);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(3);
    // ---- V: W blocks on the DMMA pipe, partial row sums ----
    for (int w = blockIdx.x; w < v_a + v_b; w += nblk) {
      const bool on_b = w >= v_a;
      const ScoreArgs& s = on_b ? g.b : g.a;
      const int q = on_b ? w - v_a : w, nvb = s.np / kVarCols;
      var_small_dispatch(s, q % nvb, q / nvb, smem);
      __syncthreads();
    }
    VZ_GT(4);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(5);
    // ---- U: scores, pool update ----
    if (blockIdx.x == 0) {
      int clamped = 0;
      const int p8 = tid & 7;
      for (int m0 = 0; m0 < e.B; m0 += kSmallThreads / 8) {
        const int m = m0 + (tid >> 3);
        const bool act = m < e.B;
        if (g.wl_a) small_finalize_8<true, GENERIC>(g.a, m, p8, act, clamped);
        else small_finalize_8<false, GENERIC>(g.a, m, p8, act, clamped);
        if (two) {
          if (g.wl_b) small_finalize_8<true, false>(g.b, m, p8, act, clamped);
          else small_finalize_8<false, false>(g.b, m, p8, act, clamped);
          __syncwarp();
          if (act && p8 == 0) {
            double acq;
            if (g.pe_mode == 0) {
              acq = fma(g.ucb, g.b.sigma[m], g.a.mu[m]);
            } else {
              const double explore_ucb = fma(g.a.sigma[m], g.explore, g.a.mu[m]);
              acq = g.b.sigma[m] + g.penalty * fmin(explore_ucb - g.threshold, 0.0);
            }
            e.batch_r[m] = tr_apply(g.tr, acq, g.wl_b ? g.b.linf[m] : INFINITY);   // b.linf: only with the distance
          }
        }
      }
      if (clamped) atomicAdd(g.a.clamp_count, clamped);
      __syncthreads();
      eagle_update_block<false>(e, smem);
    }
    VZ_GT(6);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(7);
  }
#ifdef VZ_EAGLE_TIMING
  if (tid == 0 && blockIdx.x == nblk - 1)
    printf("var_small last block: cycles/step prologue %lld wait %lld sync %lld issue %lld compute %lld\n", g_var_t[0] / g.steps,
           g_var_t[1] / g.steps, g_var_t[2] / g.steps, g_var_t[3] / g.steps, g_var_t[4] / g.steps);
  if (tid == 0 && (blockIdx.x == 0 || blockIdx.x == nblk - 1))
    printf("eagle grid cta %d/%u: cycles/step S %lld bar %lld C %lld bar %lld V %lld bar %lld U %lld bar %lld\n", (int)blockIdx.x, nblk,
           c_[0] / g.steps, c_[1] / g.steps, c_[2] / g.steps, c_[3] / g.steps, c_[4] / g.steps, c_[5] / g.steps,
           c_[6] / g.steps, c_[7] / g.steps);
#endif
}

bool eagle_grid_eligible(const vzgp_handle* h, const vzgp_handle* hB, const EagleDev& e) {
  if (e.Dk > kMaxDk) return false;   // dk x kPXLD slabs in shared memory
  static const bool enabled = [] { const char* v = getenv("VZGP_EAGLE_GRID"); return !(v && v[0] == '0'); }();
  int coop = 0;
  if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device) != cudaSuccess) coop = 0;
  const bool linear = h->kp.use_linear || (hB != nullptr && hB->kp.use_linear);   // in-kernel scoring knows Matern only
  return enabled && coop && !linear && e.B <= 8 * kTM;
}

// acq (UCB on h) or pe (GP-UCB-PE on h = model A and hB = model B): exactly one is non-null.
int launch_eagle_grid(vzgp_handle* h, vzgp_handle* hB, const EagleDev& e, const vzgp_acq* acq,
                      const vzgp_pe_params* pe, int steps, const AcqFn* fn) {
  static thread_local GridArgs G;   // several KB (descriptors, parameter tables): kept off the stack
  G.e = e;
  G.steps = steps;
  const double* xs = e.batch;
  const int32_t* zs = h->dk > 0 ? e.batch_z : nullptr;
  bool wl = false;
  if (!pe) {
    VZ_TRY(prepare_small_score(h, xs, zs, e.B, acq, e.batch_r, nullptr, nullptr, nullptr, &G.a, &wl, fn));
    G.b = G.a;
    G.pe_mode = -1; G.wl_a = wl ? 1 : 0; G.wl_b = 0;
    G.ucb = G.explore = G.penalty = G.threshold = 0.0; G.tr = TrustRegion{};
  } else {
    VZ_TRY(h->pe_tmp.reserve(sizeof(double) * 6 * (size_t)e.B));
    double* t = h->pe_tmp.as<double>();
    double* mu_a = t; double* sd_a = t + e.B; double* sd_b = t + 2 * (size_t)e.B;
    double* linf_b = t + 3 * (size_t)e.B; double* dummy_a = t + 4 * (size_t)e.B; double* dummy_b = t + 5 * (size_t)e.B;
    const vzgp_acq none = posterior_request(), accb = posterior_request(pe->tr_dim_mask, pe->tr_rows);
    G.tr = trust_region_of(hB, *pe, true);
    VZ_TRY(prepare_small_score(h, xs, zs, e.B, &none, dummy_a, mu_a, sd_a, nullptr, &G.a, &wl));
    G.wl_a = wl ? 1 : 0;
    VZ_TRY(prepare_small_score(hB, xs, zs, e.B, &accb, dummy_b, nullptr, sd_b, tr_needs_distance(G.tr) ? linf_b : nullptr,
                               &G.b, &wl));
    G.wl_b = wl ? 1 : 0;
    G.pe_mode = pe->mode; G.ucb = pe->ucb_coefficient; G.explore = pe->explore_coefficient;
    G.penalty = pe->penalty_coefficient; G.threshold = pe->threshold;
  }
  // dynamic shared memory = the largest phase
  size_t sm = eagle_suggest_cta_smem(e);
  const size_t s_u = eagle_update_smem(e), s_c = cross_small_smem_bytes(h->dc, h->dk), s_v = var_small_smem_bytes();
  if (s_u > sm) sm = s_u;
  if (s_c > sm) sm = s_c;
  if (s_v > sm) sm = s_v;
  if (sm > kMaxDynSmem) { set_error("eagle grid kernel needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
  const void* kfn = (!pe && !acq_fn_is_ucb(G.a.acq)) ? (const void*)k_eagle_grid<true> : (const void*)k_eagle_grid<false>;
  VZ_TRY(raise_dyn_smem(kfn, sm));
  int occ = 0;
  VZ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, kSmallThreads, sm));
  if (occ < 1) { set_error("eagle grid kernel does not fit on an SM"); return VZGP_ERR_UNSUPPORTED; }
  const int ntiles = (e.B + kTM - 1) / kTM;
  int want = (G.a.np / kVarCols) * ntiles + (pe ? (G.b.np / kVarCols) * ntiles : 0);   // W items >= K* items
  int grid = want < h->sm_count ? want : h->sm_count;   // one CTA per SM keeps the barrier cheap
  if (grid < 1) grid = 1;
  unsigned* bar = reinterpret_cast<unsigned*>(h->small.as<char>() + 16);   // bytes 16..19 of the small buffer
  VZ_CUDA(cudaMemsetAsync(bar, 0, sizeof(unsigned), h->stream));
  G.barrier = bar;
  void* params[] = {&G};
  VZ_CUDA(cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(kSmallThreads), params, sm, h->stream));
  h->launches++;
  return 0;
}

// ---- GP-UCB-PE over uniform ensembles ----------------------------------------------------------------------------
// The 2E member argument blocks travel in the kernel parameter (__grid_constant__, so the TMA descriptors they hold
// stay in parameter space as in k_eagle_grid).  Each ScoreArgs is about 2 KB, and the parameter space holds 32 764
// bytes, so the cooperative form takes E <= 7; E = 8 runs the replayed-graph form.
constexpr int kMaxGridPeEnsemble = 7;
struct GridEnsArgs {
  ScoreArgs m[2 * kMaxGridPeEnsemble];   // A members 0..E-1, then B members 0..E-1 (first: 64-byte aligned maps)
  EagleDev e;
  PeEnsCombine p;
  const double* mu_a;   // [E][B] member means / stddevs, written by the members' finalize
  const double* sd_a;
  const double* mu_b;
  const double* sd_b;
  const double* linf;   // [B] distance to B's trusted trials (B member 0), when the region needs it
  int n;                // 2E member models
  int wl[2 * kMaxGridPeEnsemble];                  // member computes the trust-region distance
  int c_off[2 * kMaxGridPeEnsemble + 1];           // phase C work items of members < k
  int v_off[2 * kMaxGridPeEnsemble + 1];           // phase V work items of members < k
  int steps;
  unsigned* barrier;    // zeroed by the host before the launch
};
static_assert(sizeof(GridEnsArgs) <= 32764, "the member argument blocks must fit in the kernel parameter space");

__device__ __forceinline__ int member_of(const int* off, int w) {
  int k = 0;
  while (w >= off[k + 1]) ++k;
  return k;
}

__global__ void __launch_bounds__(kSmallThreads) k_eagle_grid_pe_ensemble(const __grid_constant__ GridEnsArgs g) {
  extern __shared__ double smem[];
  const EagleDev& e = g.e;
  const int tid = threadIdx.x;
  const unsigned nblk = gridDim.x;
  unsigned gen = 0;
  const int ntiles = (e.B + kTM - 1) / kTM;
  const int rgs = ntiles == 1 ? (e.B + 15) / 16 : 4;     // 16-candidate row groups per tile
  const int n = g.n, E = g.n / 2;
  for (int it = 0; it < g.steps; ++it) {
    // ---- S: new batch ----
    for (int fb = blockIdx.x; fb < e.B; fb += nblk) eagle_suggest_cta<kSmallThreads>(e, fb, smem);
    grid_barrier(g.barrier, nblk, gen);
    // ---- C: K* blocks, partial mean / distance, over the 2E members ----
    for (int w = blockIdx.x; w < g.c_off[n]; w += nblk) {
      const int k = member_of(g.c_off, w);
      const ScoreArgs& s = g.m[k];
      const int q = w - g.c_off[k], nmb = s.np / 64;
      const int jb = q % nmb, tr = q / nmb, tile = tr / rgs, rg = tr % rgs;
      if (g.wl[k]) cross_small_block<true>(s, jb, tile, rg, smem);
      else cross_small_block<false>(s, jb, tile, rg, smem);
      __syncthreads();
    }
    grid_barrier(g.barrier, nblk, gen);
    // ---- V: W blocks on the DMMA pipe, partial row sums ----
    for (int w = blockIdx.x; w < g.v_off[n]; w += nblk) {
      const int k = member_of(g.v_off, w);
      const ScoreArgs& s = g.m[k];
      const int q = w - g.v_off[k], nvb = s.np / kVarCols;
      var_small_dispatch(s, q % nvb, q / nvb, smem);
      __syncthreads();
    }
    grid_barrier(g.barrier, nblk, gen);
    // ---- U: member moments, mixture score, pool update ----
    if (blockIdx.x == 0) {
      int clamped = 0;
      const int p8 = tid & 7;
      for (int m0 = 0; m0 < e.B; m0 += kSmallThreads / 8) {
        const int m = m0 + (tid >> 3);
        const bool act = m < e.B;
        for (int k = 0; k < n; ++k) {
          if (g.wl[k]) small_finalize_8<true, false>(g.m[k], m, p8, act, clamped);
          else small_finalize_8<false, false>(g.m[k], m, p8, act, clamped);
        }
        __syncwarp();
        if (act && p8 == 0) {   // the lane that wrote every member's moments of m reads them back
          double mean_a, s_a, mean_b, s_b;
          pe_mixture(E, g.mu_a, g.sd_a, (size_t)e.B, m, mean_a, s_a);
          pe_mixture(E, g.mu_b, g.sd_b, (size_t)e.B, m, mean_b, s_b);
          e.batch_r[m] = pe_ensemble_score(g.p, mean_a, s_a, s_b, g.wl[E] ? g.linf[m] : INFINITY);
        }
      }
      if (clamped) atomicAdd(g.m[0].clamp_count, clamped);
      __syncthreads();
      eagle_update_block<false>(e, smem);
    }
    grid_barrier(g.barrier, nblk, gen);
  }
}

bool eagle_grid_pe_ensemble_eligible(vzgp_handle* const* hAs, vzgp_handle* const* hBs, int E, const EagleDev& e) {
  if (E < 2 || E > kMaxGridPeEnsemble) return false;
  const vzgp_handle* hs[2 * kMaxGridPeEnsemble];
  for (int k = 0; k < E; ++k) { hs[k] = hAs[k]; hs[E + k] = hBs[k]; }
  for (int k = 0; k < 2 * E; ++k) {
    if (hs[k]->kp.use_linear) return false;                     // in-kernel scoring knows Matern only
    for (int j = 0; j < k; ++j)
      if (hs[j] == hs[k]) return false;                         // every member needs its own workspaces
  }
  return eagle_grid_eligible(hAs[0], hBs[0], e);
}

int launch_eagle_grid_pe_ensemble(vzgp_handle* const* hAs, vzgp_handle* const* hBs, int E, const EagleDev& e,
                                  const vzgp_pe_params* pe, int steps) {
  static thread_local GridEnsArgs G;   // ~30 KB: kept off the stack
  vzgp_handle* h = hAs[0];
  G.e = e;
  G.steps = steps;
  G.n = 2 * E;
  const int B = e.B;
  const double* xs = e.batch;
  const int32_t* zs = h->dk > 0 ? e.batch_z : nullptr;
  VZ_TRY(h->pe_tmp.reserve(sizeof(double) * (4 * (size_t)E + 2) * (size_t)B));
  double* t = h->pe_tmp.as<double>();
  double* mu_a = t;
  double* sd_a = t + (size_t)E * B;
  double* mu_b = t + 2 * (size_t)E * B;
  double* sd_b = t + 3 * (size_t)E * B;
  double* linf_b = t + 4 * (size_t)E * B;
  double* dummy = t + (4 * (size_t)E + 1) * B;
  G.mu_a = mu_a; G.sd_a = sd_a; G.mu_b = mu_b; G.sd_b = sd_b; G.linf = linf_b;
  G.p = pe_ensemble_args(hBs[0], E, pe);
  const vzgp_acq none = posterior_request(), accb = posterior_request(pe->tr_dim_mask, pe->tr_rows);
  const int ntiles = (B + kTM - 1) / kTM;
  const int rgs = ntiles == 1 ? (B + 15) / 16 : 4;
  G.c_off[0] = G.v_off[0] = 0;
  for (int k = 0; k < 2 * E; ++k) {
    const bool on_b = k >= E;
    const int me = on_b ? k - E : k;
    vzgp_handle* hk = on_b ? hBs[me] : hAs[me];
    double* mu_k = (on_b ? mu_b : mu_a) + (size_t)me * B;
    double* sd_k = (on_b ? sd_b : sd_a) + (size_t)me * B;
    const bool dist = on_b && me == 0 && tr_needs_distance(G.p.tr);
    bool wl = false;
    VZ_TRY(prepare_small_score(hk, xs, zs, B, dist ? &accb : &none, dummy, mu_k, sd_k, dist ? linf_b : nullptr,
                               &G.m[k], &wl));
    G.wl[k] = wl ? 1 : 0;
    G.c_off[k + 1] = G.c_off[k] + (hk->np / 64) * ntiles * rgs;
    G.v_off[k + 1] = G.v_off[k] + (hk->np / kVarCols) * ntiles;
  }
  size_t sm = eagle_suggest_cta_smem(e);
  const size_t s_u = eagle_update_smem(e), s_c = cross_small_smem_bytes(h->dc, h->dk), s_v = var_small_smem_bytes();
  if (s_u > sm) sm = s_u;
  if (s_c > sm) sm = s_c;
  if (s_v > sm) sm = s_v;
  if (sm > kMaxDynSmem) { set_error("eagle grid kernel needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
  const void* kfn = (const void*)k_eagle_grid_pe_ensemble;
  VZ_TRY(raise_dyn_smem(kfn, sm));
  int occ = 0;
  VZ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, kSmallThreads, sm));
  if (occ < 1) { set_error("eagle grid kernel does not fit on an SM"); return VZGP_ERR_UNSUPPORTED; }
  const int want = G.v_off[2 * E];   // W items >= K* items
  int grid = want < h->sm_count ? want : h->sm_count;   // one CTA per SM keeps the barrier cheap
  if (grid < 1) grid = 1;
  unsigned* bar = reinterpret_cast<unsigned*>(h->small.as<char>() + 16);   // bytes 16..19 of the small buffer
  VZ_CUDA(cudaMemsetAsync(bar, 0, sizeof(unsigned), h->stream));
  G.barrier = bar;
  void* params[] = {&G};
  VZ_CUDA(cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(kSmallThreads), params, sm, h->stream));
  h->launches++;
  return 0;
}

}  // namespace vzgp
