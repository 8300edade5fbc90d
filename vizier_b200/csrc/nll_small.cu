// NLL + gradient for small studies (N <= 64) in ONE kernel launch.
//
// The ARD loop (jaxopt_wrappers.py:108-199 driving stochastic_process_model.py:940-966) evaluates the
// loss a few hundred times per suggest().  For N <= 64 the general path is ~16 tiny launches and two
// host round trips per evaluation; here one CTA keeps the whole model in shared memory and runs the stages of
// nll_small.cuh; the host finishes with the regularisers.
#include "launchers.h"
#include "nll_small.cuh"

namespace vzgp {

// Without a minimum of one CTA per SM ptxas holds the wide form to 64 registers and spills.
template <bool WIDE>
__global__ void __launch_bounds__(256, WIDE ? 1 : 0) k_nll_grad_small(const double* __restrict__ X, const int32_t* __restrict__ Z,
                                                        const double* __restrict__ y, int N, int n_valid,
                                                        KernelParams kp, double sn2, double jitter0, int max_iters,
                                                        double* __restrict__ out) {
  extern __shared__ double smem[];
  __shared__ int s_bad;
  nll_small_stage<WIDE>(X, Z, y, N, n_valid, kp.dc, kp.dk, smem);
  __syncthreads();
  nll_small_eval<WIDE>(Z, N, n_valid, kp, [&](int k) { return __ldg(kp.inv_ls2_k_wide + k); }, sn2, jitter0, max_iters,
                       smem, &s_bad, out);
}

size_t nll_small_smem_bytes(int dc, int dk) {
  const int nq = dc + dk + 2;
  const int zk = dk > kMaxDk ? kCatTile : dk;
  return sizeof(double) * (4 * 64 * kSmallLD + 32 * 34 + (size_t)dc * kSmallLD + 6 * 64 + 8 * nq) + sizeof(int32_t) * (size_t)zk * kSmallLD;
}

int launch_nll_grad_small(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int n_valid,
                          const KernelParams& kp, double sn2, double jitter0, int max_iters, double* out) {
  const size_t sm = nll_small_smem_bytes(kp.dc, kp.dk);
  const auto kfn = kp.dk > kMaxDk ? k_nll_grad_small<true> : k_nll_grad_small<false>;
  VZ_TRY(raise_dyn_smem((const void*)kfn, sm));
  kfn<<<1, 256, sm, h->stream>>>(X, Z, y, N, n_valid, kp, sn2, jitter0, max_iters, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
