// The acquisition and its gradient with respect to the candidate's continuous features, for the L-BFGS-B
// acquisition optimiser (LBFGSBOptimizer, lbfgsb_optimizer.py:48-230; vzgp_score_grad / vzgp_score_grad_ensemble).
//
// Per member handle and chunk of at most kGeneralChunk candidates (DESIGN §6j):
//   1. K* and W = K* Linv^T                     launch_general_chunk (the general scoring route's two GEMMs)
//   2. V = W Linv, row m = K_y^-1 k(x_m)          k_grad_solve (only the lower-triangular blocks of Linv)
//   3. one CTA per candidate:                    k_grad_rows
//        mu = k.alpha + mean_const,  var = kss - |w|^2 + sn2 (not yet clamped),
//        dmu_d = sum_n dk_n/dx_d alpha_n,  dvar_d = dkss/dx_d - 2 sum_n dk_n/dx_d v_n,
//        and for the lead member the L-inf trust-region distance and the coordinate its gradient sits on.
//   4. after the last member, one thread per candidate:  k_grad_combine
//        the two-pass mixture of the E members (E = 1: the member itself), the acquisition, its chain rule
//        s_mu dmean + s_sd dvar / (2 sd), and the trust region: a point outside scores -1e4 - dist with
//        gradient -d dist / dx.
// Value and gradient come from the same moments, so L-BFGS-B sees a consistent pair.  Linv is read k-major rather
// than through LinvT, which only the dataflow factorisation produces.
#include "device.cuh"
#include "launchers.h"

namespace vzgp {

namespace {

using GradGemm = GemmCfg<64, 64, 16, 4, 4>;
constexpr int kRowThreads = 256;
constexpr int kMaxGradEnsemble = 16;

// V[i, j] = sum_{k >= j} W[i, k] Linv[k, j]  (W [mp x np], Linv lower [np x np], both row-major with ld np).
__global__ void __launch_bounds__(256) k_grad_solve(const double* __restrict__ W, const double* __restrict__ Linv,
                                                    int np, double* __restrict__ V) {
  extern __shared__ double smem[];
  const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
  double acc[4][4] = {};
  gemm_mainloop<64, 64, 16, 4, 4, false, true>(W, np, i0, Linv, np, j0, j0, np, acc, smem);
  const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; j += 2)
      *reinterpret_cast<double2*>(V + (size_t)(i0 + GradGemm::row_of(ty, i)) * np + j0 + GradGemm::col_of(tx, j)) =
          make_double2(acc[i][j], acc[i][j + 1]);
}

struct GradRowsArgs {
  const double* Xp;      // [mp x dc] padded candidates of this chunk
  const double* XTu;     // [dc][np] trials, unscaled, transposed
  const double* alpha;   // [np]
  double* W;             // [mp x np]; row m is overwritten with f_n = 2 dk/d(d2) (see k_grad_rows)
  const double* V;       // [mp x np]
  int np, n_valid, dc, want_linf;
  KernelParams kp;
  double sn2, mean_const;
  TrustRegion tr;
  double* mu;     // [C]      this member's planes (C = kGeneralChunk)
  double* var;    // [C]
  double* dmu;    // [C x dc]
  double* dvar;   // [C x dc]
  double* linf;   // [C] lead member only (else nullptr)
  double* trd;    // [C] signed 1 + coordinate of the distance's gradient, 0 for none
};

// Warp then block minimum of (dist, trial); ties go to the lower trial index.  Result valid in thread 0.
__device__ __forceinline__ void block_argmin(double& v, int& i, double* red_v, int* red_i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_down_sync(0xffffffffu, v, o);
    const int oi = __shfl_down_sync(0xffffffffu, i, o);
    if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) { red_v[w] = v; red_i[w] = i; }
  __syncthreads();
  if (w == 0) {
    v = lane < kRowThreads / 32 ? red_v[lane] : INFINITY;
    i = lane < kRowThreads / 32 ? red_i[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_down_sync(0xffffffffu, v, o);
      const int oi = __shfl_down_sync(0xffffffffu, i, o);
      if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
  }
}

// One CTA per candidate m.  Each thread reads w_n of row m of W and writes f_n = 2 dk_n/d(d2) in its place; the
// feature loop reads f and row m of V back from global memory (L1 / L2), so no shared-memory row limits the
// trial count.
__global__ void __launch_bounds__(kRowThreads) k_grad_rows(GradRowsArgs a) {
  __shared__ double xs[kMaxDc];
  __shared__ double red_v[32];
  __shared__ int red_i[32];
  __shared__ double s_mean, s_dist;
  __shared__ int s_best;
  const int m = blockIdx.x, tid = threadIdx.x;
  const KernelParams& kp = a.kp;
  for (int d = tid; d < a.dc; d += kRowThreads) xs[d] = a.Xp[(size_t)m * a.dc + d];
  __syncthreads();
  double* w = a.W + (size_t)m * a.np;
  const double* vrow = a.V + (size_t)m * a.np;
  double mean = 0.0, rs = 0.0, dist = INFINITY;
  int best = 0x7fffffff;
  for (int n = tid; n < a.np; n += kRowThreads) {
    const double wn = w[n];
    rs = fma(wn, wn, rs);
    double f = 0.0;
    if (n < a.n_valid) {
      // k(x, X_n) in the arithmetic of k_cross_kernel (tile_d2, tile_lin, matern52)
      double d2 = 0.0, lin = 0.0, mx = 0.0;
      for (int d = 0; d < a.dc; ++d) {
        const double xn = a.XTu[(size_t)d * a.np + n];
        const double diff = xs[d] - xn;
        d2 = fma(diff * diff, kp.inv_ls2_c[d], d2);
        if (kp.use_linear) lin = fma(fma(xs[d], kp.inv_ls_c[d], -kp.lin_b), fma(xn, kp.inv_ls_c[d], -kp.lin_b), lin);
        if (a.tr.mask[d]) mx = fmax(mx, fabs(diff));
      }
      const double s = sqrt(5.0 * d2), es = exp(-s);
      double k = kp.sf2 * (1.0 + s + s * s * (1.0 / 3.0)) * es;
      if (kp.use_linear) k = fma(kp.lin_a, lin, k);
      f = -(5.0 / 3.0) * kp.sf2 * (1.0 + s) * es;
      mean = fma(k, a.alpha[n], mean);
      if (a.want_linf && n < a.tr.rows && mx < dist) { dist = mx; best = n; }
    }
    w[n] = f;
  }
  mean = block_sum(mean, red_v);
  if (tid == 0) s_mean = mean;
  rs = block_sum(rs, red_v);
  if (tid == 0) {
    double kss = kp.sf2;
    if (kp.use_linear) {
      double uu = 0.0;
      for (int d = 0; d < a.dc; ++d) {
        const double u = fma(xs[d], kp.inv_ls_c[d], -kp.lin_b);
        uu = fma(u, u, uu);
      }
      kss = fma(kp.lin_a, uu, kss);
    }
    a.mu[m] = s_mean + a.mean_const;
    a.var[m] = kss - rs + a.sn2;
  }
  if (a.linf != nullptr) {
    block_argmin(dist, best, red_v, red_i);
    if (tid == 0) { s_dist = dist; s_best = best; }
    __syncthreads();
    if (tid == 0) {
      // d dist / dx: the first masked coordinate that attains the maximum at the nearest trial, sign(x_d - X_nd)
      double code = 0.0;
      if (s_best < a.n_valid && s_dist > 0.0 && s_dist < INFINITY) {
        for (int d = 0; d < a.dc; ++d) {
          const double diff = xs[d] - a.XTu[(size_t)d * a.np + s_best];
          if (a.tr.mask[d] && fabs(diff) == s_dist) { code = diff > 0.0 ? d + 1.0 : -(d + 1.0); break; }
        }
      }
      a.linf[m] = s_dist;
      a.trd[m] = code;
    }
  }
  __syncthreads();   // f complete in row m of W
  const int lane = tid & 31, warp = tid >> 5;
  for (int d = warp; d < a.dc; d += kRowThreads / 32) {
    const double xd = xs[d], il2 = kp.inv_ls2_c[d], il = kp.inv_ls_c[d];
    const double* xt = a.XTu + (size_t)d * a.np;
    double am = 0.0, av = 0.0;
    for (int n = lane; n < a.n_valid; n += 32) {
      const double xn = xt[n];
      double t = w[n] * (xd - xn) * il2;
      if (kp.use_linear) t = fma(kp.lin_a * il, fma(xn, il, -kp.lin_b), t);
      am = fma(t, a.alpha[n], am);
      av = fma(t, vrow[n], av);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      am += __shfl_xor_sync(0xffffffffu, am, o);
      av += __shfl_xor_sync(0xffffffffu, av, o);
    }
    if (lane == 0) {
      const double dkss = kp.use_linear ? 2.0 * kp.lin_a * fma(xd, il, -kp.lin_b) * il : 0.0;
      a.dmu[(size_t)m * a.dc + d] = am;
      a.dvar[(size_t)m * a.dc + d] = fma(-2.0, av, dkss);
    }
  }
}

// d acq_term / d mean and d acq_term / d sd, the branch acq_term evaluates.  At sd = 0 (clamped variance) EI's
// max(imp, 0) has slope [imp > 0] in the mean and PI's step has none; the stddev slope is dropped by the caller.
__device__ __forceinline__ void acq_term_slopes(const AcqTerm& t, double mean, double sd, double& s_mu, double& s_sd) {
  if (t.kind == VZGP_ACQ_LCB) { s_mu = 1.0; s_sd = -t.coefficient; return; }
  if (t.kind == VZGP_ACQ_EI || t.kind == VZGP_ACQ_PI) {
    const double imp = (mean - t.best_label) - t.exploration;
    if (!(sd > 0.0)) { s_mu = (t.kind == VZGP_ACQ_EI && imp > 0.0) ? 1.0 : 0.0; s_sd = 0.0; return; }
    const double u = imp / sd, phi = 0.3989422804014327 * exp(-0.5 * u * u);
    if (t.kind == VZGP_ACQ_EI) { s_mu = normcdf(u); s_sd = phi; return; }
    s_mu = phi / sd; s_sd = -u * phi / sd;
    return;
  }
  s_mu = 1.0; s_sd = t.coefficient;
}

struct GradCombine {
  int E, dc, have_dist;   // have_dist: the lead member wrote the distance planes
  size_t member;    // doubles between two members' planes
  AcqFn acq;
  TrustRegion tr;
};

// planes: member e at planes + e * member: mu [C], var [C], dmu [C x dc], dvar [C x dc]; then linf [C], trd [C].
__global__ void __launch_bounds__(256) k_grad_combine(int mc, GradCombine p, const double* __restrict__ planes,
                                                      double* __restrict__ score, double* __restrict__ grad,
                                                      double* __restrict__ mu, double* __restrict__ sigma,
                                                      double* __restrict__ linf, int* __restrict__ clamp_count) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= mc) return;
  constexpr size_t C = kGeneralChunk;
  const double* tail = planes + (size_t)p.E * p.member;
  double s = 0.0;
  for (int e = 0; e < p.E; ++e) s += planes[e * p.member + m];
  const double mean = s / p.E;
  double v = 0.0, q = 0.0;
  unsigned clamped = 0;
  for (int e = 0; e < p.E; ++e) {
    const double* pe = planes + e * p.member;
    double ve = pe[C + m];
    if (ve < 0.0) { ve = 0.0; clamped |= 1u << e; }
    const double dm = pe[m] - mean;
    v += ve;
    q = fma(dm, dm, q);
  }
  if (clamped) atomicAdd(clamp_count, __popc(clamped));
  const double var = v / p.E + q / p.E;
  const double sd = sqrt(var);
  const double dist = p.have_dist ? tail[m] : INFINITY;
  score[m] = tr_apply(p.tr, acq_value(p.acq, mean, sd), dist);
  if (mu) mu[m] = mean;
  if (sigma) sigma[m] = sd;
  if (linf) linf[m] = dist;
  double* g = grad + (size_t)m * p.dc;
  const bool inside = (p.tr.strict ? (dist < p.tr.radius) : (dist <= p.tr.radius)) || (p.tr.radius > 0.5);
  if (p.tr.apply && !inside) {   // tr_apply's -1e4 - dist
    const int code = (int)tail[C + m];
    for (int d = 0; d < p.dc; ++d) g[d] = 0.0;
    if (code != 0) g[(code > 0 ? code : -code) - 1] = code > 0 ? -1.0 : 1.0;
    return;
  }
  double s_mu, s_sd;
  if (p.acq.main.kind == VZGP_ACQ_MES) mes_value<true>(p.acq, mean, sd, &s_mu, &s_sd);   // sd = 0: no slope
  else acq_term_slopes(p.acq.main, mean, sd, s_mu, s_sd);
  if (p.acq.use_thr) {
    const double t = acq_term(p.acq.thr, mean, sd);
    if (!(t >= p.acq.threshold)) {   // bad_value - t
      acq_term_slopes(p.acq.thr, mean, sd, s_mu, s_sd);
      s_mu = -s_mu; s_sd = -s_sd;
    }
  }
  const double k_sd = sd > 0.0 ? s_sd / (2.0 * sd) : 0.0;
  for (int d = 0; d < p.dc; ++d) {
    double dm = 0.0, dv = 0.0, dspread = 0.0;
    for (int e = 0; e < p.E; ++e) {
      const double* pe = planes + e * p.member;
      const double dme = pe[2 * C + (size_t)m * p.dc + d];
      dm += dme;
      if (!(clamped >> e & 1u)) dv += pe[2 * C + C * p.dc + (size_t)m * p.dc + d];
      dspread = fma(pe[m] - mean, dme, dspread);
    }
    g[d] = s_mu * (dm / p.E) + k_sd * (dv / p.E + 2.0 * dspread / p.E);
  }
}

}  // namespace

int launch_score_grad(vzgp_handle* const* hs, int E, const double* Xs, int M, const vzgp_acq* acq, const AcqFn* fn,
                      double* score, double* grad, double* mu, double* sigma, double* linf) {
  if (M <= 0) return 0;
  vzgp_handle* h0 = hs[0];
  const int dc = h0->dc;
  if (E > kMaxGradEnsemble) { set_error("score_grad: at most %d members", kMaxGradEnsemble); return VZGP_ERR_ARG; }
  constexpr size_t C = kGeneralChunk;
  GradCombine p;
  p.E = E; p.dc = dc; p.member = (2 + 2 * (size_t)dc) * C;
  p.acq = acq_fn_of(acq, fn);
  p.tr = trust_region_of(h0, *acq, acq->tr_strict);
  const bool want_linf = linf != nullptr || tr_needs_distance(p.tr);
  p.have_dist = want_linf ? 1 : 0;
  VZ_TRY(h0->pe_tmp.reserve(sizeof(double) * (E * p.member + 2 * C)));
  double* planes = h0->pe_tmp.as<double>();
  for (int m0 = 0; m0 < M; m0 += (int)C) {
    const int mc = M - m0 < (int)C ? M - m0 : (int)C, mp = round_up(mc, 64);
    for (int e = 0; e < E; ++e) {
      vzgp_handle* h = hs[e];
      const int np = h->np;   // members share the valid trials, not necessarily the padded size
      GeneralChunk c;
      VZ_TRY(general_chunk_buffers(h, &c));
      VZ_TRY(launch_general_chunk(h, Xs + (size_t)m0 * dc, nullptr, mc, c));
      // V overwrites K*, which the row kernel recomputes
      k_grad_solve<<<dim3(np / 64, mp / 64), 256, GradGemm::kSmemBytes, h->stream>>>(c.W, h->Linv.as<double>(), np, c.Ks);
      VZ_CHECK_LAUNCH();
      GradRowsArgs a;
      a.Xp = c.Xp; a.XTu = h->XT.as<double>() + xt_plane(1, dc, np); a.alpha = h->alpha.as<double>();
      a.W = c.W; a.V = c.Ks;
      a.np = np; a.n_valid = h->n_valid; a.dc = dc; a.want_linf = (e == 0 && want_linf) ? 1 : 0;
      a.kp = h->kp; a.sn2 = h->sn2; a.mean_const = h->mean_const;
      a.tr = p.tr;
      double* pe = planes + e * p.member;
      a.mu = pe; a.var = pe + C; a.dmu = pe + 2 * C; a.dvar = pe + 2 * C + C * dc;
      a.linf = a.want_linf ? planes + E * p.member : nullptr;
      a.trd = planes + E * p.member + C;
      k_grad_rows<<<mc, kRowThreads, 0, h->stream>>>(a);
      VZ_CHECK_LAUNCH();
      h->launches += 2;
    }
    k_grad_combine<<<(mc + 255) / 256, 256, 0, h0->stream>>>(
        mc, p, planes, score + m0, grad + (size_t)m0 * dc, mu ? mu + m0 : nullptr, sigma ? sigma + m0 : nullptr,
        linf ? linf + m0 : nullptr, h0->small.as<int>());
    VZ_CHECK_LAUNCH();
    h0->launches++;
  }
  return 0;
}

}  // namespace vzgp
