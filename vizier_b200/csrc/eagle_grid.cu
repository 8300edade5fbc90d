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
#include "eagle_dev.cuh"
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
  if (sm > 227 * 1024) { set_error("eagle grid kernel needs %zu bytes of shared memory", sm); return VZGP_ERR_UNSUPPORTED; }
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

}  // namespace vzgp
