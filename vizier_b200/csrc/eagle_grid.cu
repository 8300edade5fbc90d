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
//   phase U  CTA 0                     fixed-order finalize, eagle_update_block
//
// k_eagle_grid scores one model with its acquisition function.  k_eagle_grid_pe_ensemble scores GP-UCB-PE over
// E >= 1 members per model (pe_ensemble.cuh; a pair of models is E = 1): phases C and V enumerate the work items of
// all 2E member models, phase U finalises every member and forms the mixture score.  The two kernels share the loop
// (eagle_grid_loop) and differ only in phase U's finalize.
#include "eagle_dev.cuh"
#include "pe_ensemble.cuh"
#include "score_small.cuh"

namespace vzgp {

struct GridArgs {
  ScoreArgs m[1];             // the model (first: 64-byte aligned maps)
  EagleDev e;
  int wl[1];                  // the model computes the trust-region distance
  int c_off[2], v_off[2];     // phase C / V work items of models < k
  int steps;
  unsigned* barrier;          // zeroed by the host before the launch
};

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

__device__ __forceinline__ int member_of(const int* off, int w) {
  int k = 0;
  while (w >= off[k + 1]) ++k;
  return k;
}

// The loop of both kernels over the n models g.m[0 .. n-1].  finalize(m, p8, act, clamped) runs in CTA 0 on the eight
// lanes p8 of candidate m (act: m < B) and leaves its score in e.batch_r[m].
template <class Args, class Finalize>
__device__ __forceinline__ void eagle_grid_loop(const Args& g, int n, Finalize finalize, double* smem) {
  const EagleDev& e = g.e;
  const int tid = threadIdx.x;
  const unsigned nblk = gridDim.x;
  unsigned gen = 0;
  const int ntiles = (e.B + kTM - 1) / kTM;
  const int rgs = ntiles == 1 ? (e.B + 15) / 16 : 4;     // 16-candidate row groups per tile
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
    // ---- C: K* blocks, partial mean / distance, over the n models ----
    for (int w = blockIdx.x; w < g.c_off[n]; w += nblk) {
      const int k = member_of(g.c_off, w);
      const ScoreArgs& s = g.m[k];
      const int q = w - g.c_off[k], nmb = s.np / 64;
      const int jb = q % nmb, tr = q / nmb, tile = tr / rgs, rg = tr % rgs;
      if (g.wl[k]) cross_small_block<true>(s, jb, tile, rg, smem);
      else cross_small_block<false>(s, jb, tile, rg, smem);
      __syncthreads();
    }
    VZ_GT(2);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(3);
    // ---- V: W blocks on the DMMA pipe, partial row sums ----
    for (int w = blockIdx.x; w < g.v_off[n]; w += nblk) {
      const int k = member_of(g.v_off, w);
      const ScoreArgs& s = g.m[k];
      const int q = w - g.v_off[k], nvb = s.np / kVarCols;
      var_small_dispatch(s, q % nvb, q / nvb, smem);
      __syncthreads();
    }
    VZ_GT(4);
    grid_barrier(g.barrier, nblk, gen);
    VZ_GT(5);
    // ---- U: scores, pool update ----
    if (blockIdx.x == 0) {
      int clamped = 0;
      for (int m0 = 0; m0 < e.B; m0 += kSmallThreads / 8) {
        const int m = m0 + (tid >> 3);
        finalize(m, tid & 7, m < e.B, clamped);
      }
      if (clamped) atomicAdd(g.m[0].clamp_count, clamped);
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
#undef VZ_GT
}

// At most one CTA per SM (launch_grid); saying so lets ptxas keep this loop in registers (no spills).
template <bool GENERIC>
__global__ void __launch_bounds__(kSmallThreads, 1) k_eagle_grid(const __grid_constant__ GridArgs g) {
  extern __shared__ double smem[];
  eagle_grid_loop(g, 1, [&](int m, int p8, bool act, int& clamped) {
    if (g.wl[0]) small_finalize_8<true, GENERIC>(g.m[0], m, p8, act, clamped);
    else small_finalize_8<false, GENERIC>(g.m[0], m, p8, act, clamped);
  }, smem);
}

__global__ void __launch_bounds__(kSmallThreads) k_eagle_grid_pe_ensemble(const __grid_constant__ GridEnsArgs g) {
  extern __shared__ double smem[];
  const int E = g.n / 2;
  eagle_grid_loop(g, g.n, [&](int m, int p8, bool act, int& clamped) {
    for (int k = 0; k < g.n; ++k) {
      if (g.wl[k]) small_finalize_8<true, false>(g.m[k], m, p8, act, clamped);
      else small_finalize_8<false, false>(g.m[k], m, p8, act, clamped);
    }
    __syncwarp();
    if (act && p8 == 0) {   // the lane that wrote every member's moments of m reads them back
      // A pair (E = 1) is its own mixture: its moments skip the mixture's divisions on phase U's critical path.
      double mean_a = g.mu_a[m], s_a = g.sd_a[m], mean_b, s_b = g.sd_b[m];
      if (E > 1) {
        pe_mixture(E, g.mu_a, g.sd_a, (size_t)g.e.B, m, mean_a, s_a);
        pe_mixture(E, g.mu_b, g.sd_b, (size_t)g.e.B, m, mean_b, s_b);
      }
      g.e.batch_r[m] = pe_ensemble_score(g.p, mean_a, s_a, s_b, g.wl[E] ? g.linf[m] : INFINITY);
    }
  }, smem);
}

bool eagle_grid_eligible(const vzgp_handle* h, const EagleDev& e) {
  if (e.Dk > kMaxDk) return false;   // dk x kPXLD slabs in shared memory
  static const bool enabled = [] { const char* v = getenv("VZGP_EAGLE_GRID"); return !(v && v[0] == '0'); }();
  int coop = 0;
  if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device) != cudaSuccess) coop = 0;
  return enabled && coop && !h->kp.use_linear && e.B <= 8 * kTM;   // in-kernel scoring knows Matern only
}

bool eagle_grid_pe_ensemble_eligible(vzgp_handle* const* hAs, vzgp_handle* const* hBs, int E, const EagleDev& e) {
  if (E < 1 || E > kMaxGridPeEnsemble) return false;
  const vzgp_handle* hs[2 * kMaxGridPeEnsemble];
  for (int k = 0; k < E; ++k) { hs[k] = hAs[k]; hs[E + k] = hBs[k]; }
  for (int k = 0; k < 2 * E; ++k) {
    if (hs[k]->kp.use_linear) return false;                     // in-kernel scoring knows Matern only
    for (int j = 0; j < k; ++j)
      if (hs[j] == hs[k]) return false;                         // every member needs its own workspaces
  }
  return eagle_grid_eligible(hAs[0], e);
}

// Model k of the loop on the batch of e: its argument block, and its phase C / V work items after those of models < k.
template <class Args>
static int add_grid_model(Args& g, int k, vzgp_handle* hk, const vzgp_acq* acq, double* score, double* mu, double* sd,
                          double* linf, const AcqFn* fn = nullptr) {
  const EagleDev& e = g.e;
  bool wl = false;
  VZ_TRY(prepare_small_score(hk, e.batch, e.Dk > 0 ? e.batch_z : nullptr, e.B, acq, score, mu, sd, linf, &g.m[k], &wl, fn));
  g.wl[k] = wl ? 1 : 0;
  const int ntiles = (e.B + kTM - 1) / kTM;
  const int rgs = ntiles == 1 ? (e.B + 15) / 16 : 4;
  if (k == 0) g.c_off[0] = g.v_off[0] = 0;
  g.c_off[k + 1] = g.c_off[k] + (hk->np / 64) * ntiles * rgs;
  g.v_off[k + 1] = g.v_off[k] + (hk->np / kVarCols) * ntiles;
  return 0;
}

// The cooperative launch of kernel kfn over the n models of g (h: model 0).  Dynamic shared memory is the largest
// phase's; the grid is one CTA per phase V work item (there are no fewer than phase C's), at most one per SM.
template <class Args>
static int launch_grid(vzgp_handle* h, const void* kfn, Args& g, int n) {
  size_t sm = eagle_suggest_cta_smem(g.e);
  const size_t s_u = eagle_update_smem(g.e), s_c = cross_small_smem_bytes(h->dc, h->dk), s_v = var_small_smem_bytes();
  if (s_u > sm) sm = s_u;
  if (s_c > sm) sm = s_c;
  if (s_v > sm) sm = s_v;
  if (sm > kMaxDynSmem) { set_error("eagle grid kernel needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
  VZ_TRY(raise_dyn_smem(kfn, sm));
  int occ = 0;
  VZ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, kSmallThreads, sm));
  if (occ < 1) { set_error("eagle grid kernel does not fit on an SM"); return VZGP_ERR_UNSUPPORTED; }
  const int want = g.v_off[n];
  int grid = want < h->sm_count ? want : h->sm_count;   // one CTA per SM keeps the barrier cheap
  if (grid < 1) grid = 1;
  unsigned* bar = reinterpret_cast<unsigned*>(h->small.as<char>() + 16);   // bytes 16..19 of the small buffer
  VZ_CUDA(cudaMemsetAsync(bar, 0, sizeof(unsigned), h->stream));
  g.barrier = bar;
  void* params[] = {&g};
  VZ_CUDA(cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(kSmallThreads), params, sm, h->stream));
  h->launches++;
  return 0;
}

int launch_eagle_grid(vzgp_handle* h, const EagleDev& e, const vzgp_acq* acq, int steps, const AcqFn* fn) {
  static thread_local GridArgs G;   // several KB (descriptors, parameter tables): kept off the stack
  G.e = e;
  G.steps = steps;
  VZ_TRY(add_grid_model(G, 0, h, acq, e.batch_r, nullptr, nullptr, nullptr, fn));
  const void* kfn = acq_fn_is_ucb(G.m[0].acq) ? (const void*)k_eagle_grid<false> : (const void*)k_eagle_grid<true>;
  return launch_grid(h, kfn, G, 1);
}

int launch_eagle_grid_pe_ensemble(vzgp_handle* const* hAs, vzgp_handle* const* hBs, int E, const EagleDev& e,
                                  const vzgp_pe_params* pe, int steps) {
  static thread_local GridEnsArgs G;   // ~30 KB: kept off the stack
  vzgp_handle* h = hAs[0];
  G.e = e;
  G.steps = steps;
  G.n = 2 * E;
  const int B = e.B;
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
  for (int k = 0; k < 2 * E; ++k) {
    const bool on_b = k >= E;
    const int me = on_b ? k - E : k;
    double* mu_k = on_b && E == 1 ? nullptr : (on_b ? mu_b : mu_a) + (size_t)me * B;   // a pair needs no mean of B
    double* sd_k = (on_b ? sd_b : sd_a) + (size_t)me * B;
    const bool dist = on_b && me == 0 && tr_needs_distance(G.p.tr);
    VZ_TRY(add_grid_model(G, k, on_b ? hBs[me] : hAs[me], dist ? &accb : &none, dummy, mu_k, sd_k,
                          dist ? linf_b : nullptr));
  }
  return launch_grid(h, (const void*)k_eagle_grid_pe_ensemble, G, 2 * E);
}

}  // namespace vzgp
