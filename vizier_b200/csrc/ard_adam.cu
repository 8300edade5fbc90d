// ARD with Adam (the reference's OptaxTrain, optax_wrappers.py:36-150) for small studies (N <= 64): every epoch of
// every restart in ONE launch, one CTA of 256 threads per restart.  Each CTA stages the trials once and then loops
// its epochs with no host round trip:
//   1. theta = SoftClip(u) per parameter (tuned_gp_models.py:150-270; hinge softness 1e-2) and its derivative;
//   2. the KernelParams of theta, built in shared memory;
//   3. one NLL + gradient evaluation: the stages of k_nll_grad_small (nll_small.cuh), jitter retry included;
//   4. the host-side finishing of vzgp_nll_grad_multi (c_abi.cu finish_loss: 2 pi term, regularisers) in the same
//      order of operations;
//   5. the chain rule through SoftClip;
//   6. optax's Adam update (scale_by_adam, then scale by -learning_rate).
// The elementwise arithmetic of steps 1 and 4-6 is written with explicitly rounded intrinsics (no FMA contraction),
// so it performs the IEEE operations of the NumPy restatement (tests/adam_oracle.py) and of the host-stepped route
// (vizier_b200/ard.py) one for one; only exp / log / log1p / expm1 may differ in the last bit.
// A restart whose evaluation has exhausted the jitter retries, or whose loss or gradient is not finite, stops: its
// loss is NaN from that epoch on and its parameters stay where that evaluation saw them.
#include <math_constants.h>

#include <cfloat>

#include "launchers.h"
#include "nll_small.cuh"

namespace vzgp {
namespace {

constexpr double kHinge = 1e-2;   // SoftClip hinge softness
constexpr int kJitterRetries = 5;
constexpr double kJitter0 = 1e-4;

struct AdamArgs {
  double lr, b1, b2, eps, eps_root;
  int epochs;
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// c log1p(exp(v / c)) in the overflow-free form max(v, 0) + c log1p(exp(-|v| / c)).
__device__ __forceinline__ double softplus_h(double v) {
  return dadd(fmax(v, 0.0), dmul(kHinge, log1p(exp(ddiv(-fabs(v), kHinge)))));
}
// Its inverse for s > 0: s + c log(-expm1(-s / c)).
__device__ __forceinline__ double softplus_h_inv(double s) {
  return dadd(s, dmul(kHinge, log(-expm1(ddiv(-s, kHinge)))));
}
__device__ __forceinline__ double sigmoid(double z) {
  if (z >= 0.0) return ddiv(1.0, dadd(1.0, exp(-z)));
  const double e = exp(z);
  return ddiv(e, dadd(1.0, e));
}
// y = hi - sp(hi - lo - sp(u - lo)) and dy/du = sigmoid(w / c) sigmoid((u - lo) / c), w = hi - lo - sp(u - lo).
__device__ __forceinline__ double soft_clip(double u, double lo, double hi, double* dy) {
  const double a = dsub(u, lo);
  const double w = dsub(dsub(hi, lo), softplus_h(a));
  *dy = dmul(sigmoid(ddiv(w, kHinge)), sigmoid(ddiv(a, kHinge)));
  return dsub(hi, softplus_h(w));
}
// u = lo + sp^-1(hi - lo - sp^-1(hi - y)); both arguments of sp^-1 are kept >= DBL_MIN, so a point on (or past) a
// bound maps to a finite u.
__device__ __forceinline__ double soft_clip_inv(double y, double lo, double hi) {
  const double r = softplus_h_inv(fmax(dsub(hi, y), DBL_MIN));
  return dadd(lo, softplus_h_inv(fmax(dsub(dsub(hi, lo), r), DBL_MIN)));
}
// The regulariser 0.01 log(x / c)^2 and its derivative 0.02 log(x / c) / x (tuned_gp_models.py:167,180,192,269).
__device__ __forceinline__ double reg(double x, double c) {
  const double l = log(ddiv(x, c));
  return dmul(dmul(0.01, l), l);
}
__device__ __forceinline__ double dreg(double x, double c) { return ddiv(dmul(0.02, log(ddiv(x, c))), x); }

}  // namespace

// Doubles of dynamic shared memory past the evaluation's layout: the raw sums [4 + P], per parameter u, mu, nu,
// theta, dtheta/du, dloss/dtheta, regulariser, lower and upper bound [9 P], the wide categorical weights [Dk] and the
// loss [1]; then the KernelParams of the epoch and two flags (pivot failed, non-finite gradient).
static size_t adam_extra_doubles(int dc, int dk) {
  const int p = dc + dk + 2;
  return 4 + (size_t)p + 9 * (size_t)p + (dk > kMaxDk ? (size_t)dk : 0) + 1;
}

// The kernel declares no static shared memory: everything it uses is in this count, which is therefore the whole of
// what a launch needs (tests/test_ard_adam_ptxas.py pins the 0 bytes of static shared memory ptxas reports).
size_t ard_adam_small_smem_bytes(int dc, int dk) {
  static_assert(sizeof(KernelParams) % sizeof(double) == 0, "the flags follow KernelParams at 8-byte alignment");
  return nll_small_smem_bytes(dc, dk) + sizeof(double) * adam_extra_doubles(dc, dk) + sizeof(KernelParams) +
         2 * sizeof(int);
}

// theta0, theta_out [R x P] and bounds [P] in the vzgp_nll_grad gradient order (categorical ls2, continuous ls2, noise,
// signal); loss_out, status_out [R]; trace [epochs x R] or null.
template <bool WIDE>
__global__ void __launch_bounds__(256, WIDE ? 1 : 0) k_ard_adam_small(
    const double* __restrict__ X, const int32_t* __restrict__ Z, const double* __restrict__ y, int N, int n_valid,
    int dc, int dk, int R, const double* __restrict__ theta0, const double* __restrict__ lower,
    const double* __restrict__ upper, AdamArgs adam, double* __restrict__ theta_out, double* __restrict__ loss_out,
    int* __restrict__ status_out, double* __restrict__ trace) {
  extern __shared__ double smem[];
  const int tid = threadIdx.x, r = blockIdx.x;
  const int P = dc + dk + 2, o = dk + dc;
  const SmallNllSmem lay(smem, dc, P);
  double* raw = lay.end(WIDE ? kCatTile : dk);
  double* s_u = raw + 4 + P;
  double* s_mu = s_u + P;
  double* s_nu = s_mu + P;
  double* s_th = s_nu + P;
  double* s_dth = s_th + P;
  double* s_g = s_dth + P;
  double* s_reg = s_g + P;
  double* s_lo = s_reg + P;
  double* s_hi = s_lo + P;
  double* s_wk = s_hi + P;   // WIDE: [dk]
  double& s_loss = s_wk[WIDE ? dk : 0];
  KernelParams& skp = *reinterpret_cast<KernelParams*>(&s_loss + 1);
  int* s_bad = reinterpret_cast<int*>(&skp + 1);
  int& s_nonfinite = s_bad[1];

  for (int p = tid; p < P; p += 256) {
    const double lo = lower[p], hi = upper[p];
    s_lo[p] = lo; s_hi[p] = hi;
    s_u[p] = soft_clip_inv(theta0[(size_t)r * P + p], lo, hi);
    s_mu[p] = 0.0; s_nu[p] = 0.0;
  }
  if (tid == 0) {
    skp.dc = dc; skp.dk = dk; skp.inv_ls2_k_wide = nullptr; skp.use_linear = 0; skp.lin_a = 0.0; skp.lin_b = 0.0;
  }
  nll_small_stage<WIDE>(X, Z, y, N, n_valid, dc, dk, smem);
  const double one_b1 = 1.0 - adam.b1, one_b2 = 1.0 - adam.b2, neg_lr = -adam.lr;
  const double two_pi_term = dmul(dmul(0.5, (double)n_valid), log(2.0 * M_PI));
  double b1t = 1.0, b2t = 1.0;
  int retries = 0;
  __syncthreads();
  int epoch = 0;
  for (; epoch < adam.epochs; ++epoch) {
    // ---- 1-2. theta, dtheta/du, regulariser terms, KernelParams ----
    for (int p = tid; p < P; p += 256) {
      double d;
      const double th = soft_clip(s_u[p], s_lo[p], s_hi[p], &d);
      s_th[p] = th; s_dth[p] = d;
      s_reg[p] = reg(th, p < o ? 0.5 : (p == o ? 0.0039 : 0.039));
      const double inv = 1.0 / th;
      if (p < dk) {
        if (WIDE) s_wk[p] = inv;
        else skp.inv_ls2_k[p] = inv;
      } else if (p < o) {
        skp.inv_ls2_c[p - dk] = inv;
      } else if (p == o + 1) {
        skp.sf2 = th;
      }
    }
    if (tid == 0) s_nonfinite = 0;
    __syncthreads();
    // ---- 3. one evaluation ----
    nll_small_eval<WIDE>(Z, N, n_valid, skp, [&](int k) { return s_wk[k]; }, s_th[o], kJitter0, kJitterRetries, smem,
                         s_bad, raw);
    __syncthreads();
    // ---- 4-5. loss and gradient (finish_loss), chain rule ----
    const double sn2 = s_th[o], sf2 = s_th[o + 1];
    for (int p = tid; p < P; p += 256) {
      const double th = s_th[p], gs = raw[4 + p];
      double g;
      if (p < o) g = dadd(ddiv(dmul(-0.5, gs), dmul(th, th)), dreg(th, 0.5));
      else if (p == o) g = dadd(dmul(0.5, gs), dreg(sn2, 0.0039));
      else g = dadd(ddiv(dmul(0.5, gs), sf2), dreg(sf2, 0.039));
      if (!isfinite(g)) s_nonfinite = 1;
      s_g[p] = dmul(g, s_dth[p]);
    }
    if (tid == 0) {
      double loss = dadd(dadd(raw[0], raw[1]), two_pi_term);
      loss = dadd(loss, dadd(s_reg[o + 1], s_reg[o]));
      for (int p = 0; p < o; ++p) loss = dadd(loss, s_reg[p]);
      s_loss = loss;
    }
    __syncthreads();
    retries = (int)raw[3];
    const bool stop = retries > kJitterRetries || !isfinite(s_loss) || s_nonfinite;
    if (tid == 0 && trace) trace[(size_t)epoch * R + r] = stop ? CUDART_NAN : s_loss;
    if (stop) break;
    // ---- 6. Adam ----
    b1t = dmul(b1t, adam.b1);
    b2t = dmul(b2t, adam.b2);
    const double c1 = dsub(1.0, b1t), c2 = dsub(1.0, b2t);
    for (int p = tid; p < P; p += 256) {
      const double g = s_g[p];
      const double mu = dadd(dmul(one_b1, g), dmul(adam.b1, s_mu[p]));
      const double nu = dadd(dmul(one_b2, dmul(g, g)), dmul(adam.b2, s_nu[p]));
      s_mu[p] = mu; s_nu[p] = nu;
      const double upd = ddiv(ddiv(mu, c1), dadd(__dsqrt_rn(dadd(ddiv(nu, c2), adam.eps_root)), adam.eps));
      s_u[p] = dadd(s_u[p], dmul(neg_lr, upd));
    }
    __syncthreads();
  }
  const bool stopped = epoch < adam.epochs;
  if (tid == 0) {
    loss_out[r] = stopped ? CUDART_NAN : s_loss;
    status_out[r] = retries;
    if (trace)
      for (int e = epoch + 1; e < adam.epochs; ++e) trace[(size_t)e * R + r] = CUDART_NAN;
  }
  // the parameters after the last update; a stopped restart keeps those of its last evaluation
  for (int p = tid; p < P; p += 256) {
    double d;
    theta_out[(size_t)r * P + p] = stopped ? s_th[p] : soft_clip(s_u[p], s_lo[p], s_hi[p], &d);
  }
}

int launch_ard_adam_small(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int n_valid,
                          int dc, int dk, int R, const double* theta0, const double* lower, const double* upper,
                          double lr, double b1, double b2, double eps, double eps_root, int epochs, double* theta_out,
                          double* loss_out, int* status_out, double* trace) {
  const size_t sm = ard_adam_small_smem_bytes(dc, dk);
  const auto kfn = dk > kMaxDk ? k_ard_adam_small<true> : k_ard_adam_small<false>;
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  const AdamArgs args{lr, b1, b2, eps, eps_root, epochs};
  kfn<<<R, 256, sm, h->stream>>>(X, Z, y, N, n_valid, dc, dk, R, theta0, lower, upper, args, theta_out, loss_out,
                                 status_out, trace);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
