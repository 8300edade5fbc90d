// extern "C" surface of libvzgp.so (see include/vzgp.h for the contract of each entry point).
#include <climits>
#include <cstdarg>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "launchers.h"

namespace vzgp {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int raise_dyn_smem(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> limits;
  int dev = 0;
  VZ_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = limits[{dev, kernel}];
  if (bytes <= cur) return 0;
  VZ_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  cur = bytes;
  return 0;
}

// Layout of handle->small (device, 64 KiB).
constexpr size_t kSmallBytes = 65536;
constexpr size_t kOffClamp = 0;      // int
constexpr size_t kOffFlag = 8;       // int
constexpr size_t kOffLogdet = 64;    // double[3]: M sum log L_ii, quadratic form / 2, sum alpha
constexpr size_t kOffGrad = 5120;    // double[<= 2 kMaxDc + kMaxDk + 8] (the free 3 KiB below kOffPartial)
constexpr int kMaxGrad = 2 * kMaxDc + kMaxDk + 8;
constexpr size_t kOffTopIdx = 1024;  // long long[256]
constexpr size_t kOffTopVal = 3072;  // double[256]
constexpr size_t kOffPartial = 8192; // ArgMax[<=2048] = 32 KiB
constexpr size_t kOffRows = 40960;   // winner rows of the fused top-k calls (24 KiB)
constexpr size_t kRowsBytes = kSmallBytes - kOffRows;
constexpr int kMaxTopk = 256;

struct Guard {
  int prev = -1;
  explicit Guard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~Guard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

static int ensure_model_buffers(vzgp_handle* h, int np, int dc, int dk, int n_metrics = 1) {
  VZ_TRY(h->X.reserve(sizeof(double) * (size_t)np * (dc > 0 ? dc : 1)));
  VZ_TRY(h->XT.reserve(sizeof(double) * 2 * (size_t)np * (dc > 0 ? dc : 1)));
  VZ_TRY(h->Z.reserve(sizeof(int32_t) * (size_t)np * (dk > 0 ? dk : 1)));
  VZ_TRY(h->L.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(h->Linv.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(h->LinvT.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(h->Kws.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(h->alpha.reserve(sizeof(double) * (size_t)np * n_metrics));             // [M][np]
  VZ_TRY(h->ypad.reserve(sizeof(double) * (size_t)np * 4 * n_metrics));  // [M][y, w, r, tmp]
  return 0;
}

// Factor the (already shifted) lower matrix in L in place and form L^-1.  With LinvT != nullptr the dataflow
// kernel (dataflow.cu) does both - plus L^-T and, if Kinv != nullptr, the lower tiles of L^-T L^-1 - in one
// launch; *used_dataflow tells the caller which form of Kinv exists.  Otherwise (stage-wise entry points,
// VZGP_DATAFLOW=0, a single 64-block): the panel kernels of linalg.cu + recursive doubling.
static int factor_invert(vzgp_handle* h, double* L, double* Linv, double* LinvT, double* Kinv, int np, int* flag,
                         bool* used_dataflow) {
  *used_dataflow = false;
  if (LinvT != nullptr) {
    const int st = chol_dataflow(h, L, Linv, LinvT, Kinv, np, flag);
    if (st < 0) return st;
    if (st == 0) { *used_dataflow = true; h->factor_route = VZGP_FACTOR_DATAFLOW; return 0; }
  }
  h->factor_route = VZGP_FACTOR_PANEL;
  VZ_TRY(potrf_blocked(h, L, np, Linv, np, np, flag));
  VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)np * np));
  VZ_TRY(trtri_doubling(h, L, np, Linv, np, h->Tws.as<double>(), np, np));
  return 0;
}

// Factor A (np x np device, lower read) into h-independent buffers with retry semantics.
// L, Linv: [np x np] (Linv complete on return).  Returns retries, or max_iters+1 on final failure, or <0.
static int cholesky_retry_padded(vzgp_handle* h, const double* A, int lda, int n_src, int np,
                                 double jitter0, int max_iters, double* L, double* Linv,
                                 double* shift_out, double* LinvT = nullptr, bool* used_dataflow = nullptr) {
  int* flag = reinterpret_cast<int*>(h->small.as<char>() + kOffFlag);
  double shift = 0.0;
  int attempt = 0;
  for (;;) {
    VZ_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), h->stream));
    VZ_CUDA(cudaMemsetAsync(Linv, 0, sizeof(double) * (size_t)np * np, h->stream));
    VZ_TRY(launch_copy_lower_shift(h, A, lda, n_src, np, shift, L, np));
    bool df = false;
    VZ_TRY(factor_invert(h, L, Linv, LinvT, nullptr, np, flag, &df));
    int bad = 0;
    VZ_CUDA(cudaMemcpyAsync(&bad, flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    VZ_CUDA(cudaStreamSynchronize(h->stream));
    if (df) {
      int to = 0;
      VZ_TRY(chol_dataflow_timed_out(h, &to));
      if (to) { set_error("dataflow factorisation: a tile wait timed out"); return VZGP_ERR_CUDA; }
    }
    if (used_dataflow) *used_dataflow = df;
    if (!bad) break;
    if (attempt >= max_iters) {
      if (shift_out) *shift_out = shift;
      return max_iters + 1;
    }
    shift = (shift == 0.0) ? jitter0 : shift * 10.0;
    ++attempt;
  }
  if (shift_out) *shift_out = shift;
  return attempt;
}

// alpha_m = Linv^T (Linv y_m) plus one step of iterative refinement against K_y (+shift), for every metric
// (the independent multi-task GP shares the factor: tuned_gp_models.py:282-288).  y is metric-major
// [M][N] device; ypad is [M][4][np] (y, w = Linv y, r, tmp), alpha [M][np].
static int solve_alphas(vzgp_handle* h, const double* y, int N, int n_valid, int np, int n_metrics, double shift,
                        bool have_linvT) {
  // Linv^T v: a row-wise product with L^-T when the dataflow factorisation produced it (coalesced rows)
  auto gemv_T = [&](const double* v, double* out) -> int {
    if (have_linvT) return launch_gemv_rows(h, h->LinvT.as<double>(), np, np, v, out, 2);
    return launch_gemv_lower_T(h, h->Linv.as<double>(), np, np, v, out);
  };
  for (int m = 0; m < n_metrics; ++m) {
    double* yp = h->ypad.as<double>() + (size_t)m * 4 * np;
    double* w = yp + np;
    double* r = yp + 2 * np;
    double* tmp = yp + 3 * np;
    double* alpha = h->alpha.as<double>() + (size_t)m * np;
    VZ_TRY(launch_pad_vector(h, y + (size_t)m * N, N, n_valid, np, yp, h->mean_const));
    VZ_TRY(launch_gemv_rows(h, h->Linv.as<double>(), np, np, yp, w, 1));
    VZ_TRY(gemv_T(w, alpha));
    VZ_TRY(launch_residual(h, h->Kws.as<double>(), np, np, yp, alpha, r));
    if (shift != 0.0) VZ_TRY(launch_axpy(h, np, -shift, alpha, r));
    VZ_TRY(launch_gemv_rows(h, h->Linv.as<double>(), np, np, r, tmp, 1));
    VZ_TRY(gemv_T(tmp, r));
    VZ_TRY(launch_axpy(h, np, 1.0, r, alpha));
  }
  return 0;
}

// Shared front half of fit / nll_grad: pads inputs, builds K_y, factors, inverts, solves alpha.
// On return: h->X/Z padded copies, Kws = K_y (unshifted), L, Linv, alpha valid; ypad[0..np) = y,
// ypad[np..2np) = w = Linv y.
static int fit_common(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N,
                      int dc, int dk, int n_valid, const vzgp_params* p, double* shift_used, int n_metrics = 1) {
  VZ_ARG(h != nullptr, "handle");
  VZ_ARG(N >= 1, "N >= 1");
  VZ_ARG(n_valid >= 1 && n_valid <= N, "1 <= n_valid <= N");
  VZ_ARG(n_metrics >= 1 && n_metrics <= kMaxMetrics, "1 <= n_metrics <= 8");
  VZ_ARG(X != nullptr || dc == 0, "X");
  VZ_ARG(Z != nullptr || dk == 0, "Z");
  VZ_ARG(y != nullptr, "y");
  KernelParams kp;
  VZ_TRY(fill_kernel_params(p, dc, dk, &kp));
  const int np = round_up(N, kBlk);
  VZ_TRY(ensure_model_buffers(h, np, dc, dk, n_metrics));
  h->fitted = false; h->i8_ready = false;
  h->n = N; h->np = np; h->dc = dc; h->dk = dk; h->n_valid = n_valid; h->n_metrics = n_metrics;
  h->kp = kp; h->sn2 = p->observation_noise_variance;
  h->mean_const = p->linear_coef != 0.0 ? p->linear_coef * p->mean_constant : 0.0;
  VZ_ARG(!kp.use_linear || n_metrics == 1, "linear_coef with several metrics is not implemented");
  if (dc > 0) VZ_TRY(launch_pad_rows(h, X, N, dc, np, h->X.as<double>()));
  if (dc > 0) VZ_TRY(launch_transpose_scale(h, h->X.as<double>(), np, dc, kp, h->XT.as<double>()));
  if (dk > 0) VZ_TRY(launch_pad_rows_i32(h, Z, N, dk, np, h->Z.as<int32_t>()));
  VZ_TRY(launch_kernel_matrix(h, h->X.as<double>(), h->Z.as<int32_t>(), np, n_valid, kp, h->sn2,
                              h->Kws.as<double>(), np));
  double shift = 0.0;
  bool df = false;
  int retries = cholesky_retry_padded(h, h->Kws.as<double>(), np, np, np, 1e-4, 5,
                                      h->L.as<double>(), h->Linv.as<double>(), &shift, h->LinvT.as<double>(), &df);
  if (retries < 0) return retries;
  if (shift_used) *shift_used = shift;
  VZ_TRY(solve_alphas(h, y, N, n_valid, np, n_metrics, shift, df));
  return retries;
}

// ---------------------------------------------------------------------------
// One NLL + gradient evaluation as a replayed CUDA graph (N > 64).
// The launch sequence is the one of fit_common + the gradient part with a single factorisation attempt
// and no host round trip; if the factorisation flags a bad pivot the caller falls back to the eager
// path with its retry loop.  ~50 launches per evaluation cost more host time than GPU time when several
// ARD restarts launch from different threads (the driver serialises them); replaying one graph does not.
// ---------------------------------------------------------------------------
static int nll_sequence(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int dc, int dk,
                        int n_valid, const KernelParams& kp, double sn2, int n_metrics) {
  const int np = h->np;
  int* flag = reinterpret_cast<int*>(h->small.as<char>() + kOffFlag);
  if (dc > 0) VZ_TRY(launch_pad_rows(h, X, N, dc, np, h->X.as<double>()));
  if (dc > 0) VZ_TRY(launch_transpose_scale(h, h->X.as<double>(), np, dc, kp, h->XT.as<double>()));
  if (dk > 0) VZ_TRY(launch_pad_rows_i32(h, Z, N, dk, np, h->Z.as<int32_t>()));
  VZ_TRY(launch_kernel_matrix(h, h->X.as<double>(), h->Z.as<int32_t>(), np, n_valid, kp, sn2, h->Kws.as<double>(), np));
  VZ_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), h->stream));
  VZ_CUDA(cudaMemsetAsync(h->Linv.as<double>(), 0, sizeof(double) * (size_t)np * np, h->stream));
  VZ_TRY(launch_copy_lower_shift(h, h->Kws.as<double>(), np, np, np, 0.0, h->L.as<double>(), np));
  bool df = false;   // dataflow kernel: factor, both inverses and K_y^-1 (one plane) in one launch
  VZ_TRY(factor_invert(h, h->L.as<double>(), h->Linv.as<double>(), h->LinvT.as<double>(), h->Kinv.as<double>(), np, flag, &df));
  h->nll_factor_route = h->factor_route;
  VZ_TRY(solve_alphas(h, y, N, n_valid, np, n_metrics, 0.0, df));
  double* out2 = reinterpret_cast<double*>(h->small.as<char>() + kOffLogdet);
  double* gout = reinterpret_cast<double*>(h->small.as<char>() + kOffGrad);
  VZ_TRY(launch_logdet_quad(h, h->L.as<double>(), np, N, n_valid, h->ypad.as<double>() + np, out2, 4 * np, n_metrics));
  if (!df) VZ_TRY(launch_lauum(h, h->Linv.as<double>(), np, h->Kinv.as<double>(), np, np));
  VZ_TRY(launch_nll_grad_tiles(h, h->X.as<double>(), h->Z.as<int32_t>(), np, n_valid, kp, h->Kinv.as<double>(), np,
                               h->alpha.as<double>(), h->Tws.as<double>(), gout, df ? np : 0, n_metrics));
  return 0;
}

static void nll_graph_drop(vzgp_handle* h) {
  if (h->nll_exec) cudaGraphExecDestroy(h->nll_exec);
  if (h->nll_graph) cudaGraphDestroy(h->nll_graph);
  h->nll_exec = nullptr; h->nll_graph = nullptr;
  h->nll_nodes[0] = h->nll_nodes[1] = h->nll_nodes[2] = nullptr;
}

// Returns 0 and fills host2 / hostg on success; 1 if the caller must use the eager path (bad pivot or
// the graph could not be built); < 0 on errors.
static int nll_graph_eval(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int dc, int dk,
                          int n_valid, int n_metrics, const vzgp_params* p, double* host2, double* hostg) {
  static const bool enabled = [] { const char* e = getenv("VZGP_NLL_GRAPH"); return !(e && e[0] == '0'); }();
  if (!enabled) return 1;
  KernelParams kp;
  VZ_TRY(fill_kernel_params(p, dc, dk, &kp));
  double sn2 = p->observation_noise_variance;
  const int np = round_up(N, kBlk), nq = dc + dk + 2;
  auto bufs = [&](const void** o) {
    const DevBuf* b[kNllBufs] = {&h->X, &h->XT, &h->Z, &h->L, &h->Linv, &h->alpha, &h->ypad, &h->Kws, &h->Tws, &h->Kinv, &h->small,
                                 &h->LinvT, &h->df_tasks[1], &h->df_flags, &h->df_S};
    for (int q = 0; q < kNllBufs; ++q) o[q] = b[q]->ptr;
  };
  const void* cur[kNllBufs];
  bufs(cur);
  bool hit = h->nll_exec && h->nll_key[0] == X && h->nll_key[1] == Z && h->nll_key[2] == y &&
             h->nll_key_dims[0] == N && h->nll_key_dims[1] == dc && h->nll_key_dims[2] == dk &&
             h->nll_key_dims[3] == n_valid && h->nll_key_dims[4] == n_metrics;
  hit = hit && (h->df_nb[1] == 0 || h->df_nb[1] == np / 64);   // another call re-planned the dataflow tasks
  for (int q = 0; hit && q < kNllBufs; ++q) hit = cur[q] == h->nll_bufs[q];   // a workspace was reallocated since the capture
  h->fitted = false; h->i8_ready = false;
  if (!hit) {
    nll_graph_drop(h);
    VZ_TRY(ensure_model_buffers(h, np, dc, dk, n_metrics));
    VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * kLauumSplit));
    VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)np * np));
    VZ_TRY(chol_dataflow_prepare(h, np, true));   // task list + flags: not capturable
    bufs(cur);
    h->n = N; h->np = np; h->dc = dc; h->dk = dk; h->n_valid = n_valid; h->n_metrics = n_metrics;
    h->mean_const = 0.0;   // the label-padding node captures it: a linear_coef fit before must not leak its prior mean in
    const int64_t l0 = h->launches;
    if (cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) { cudaGetLastError(); return 1; }
    const int st = nll_sequence(h, X, Z, y, N, dc, dk, n_valid, kp, sn2, n_metrics);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
    h->nll_launches = (int)(h->launches - l0);
    h->launches = l0;
    if (st < 0 || ce != cudaSuccess || !graph) { if (graph) cudaGraphDestroy(graph); cudaGetLastError(); return st < 0 ? st : 1; }
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) { cudaGraphDestroy(graph); cudaGetLastError(); return 1; }
    size_t nn = 0;
    cudaGraphGetNodes(graph, nullptr, &nn);
    std::vector<cudaGraphNode_t> nodes(nn);
    cudaGraphGetNodes(graph, nodes.data(), &nn);
    const void* want[3] = {kernel_matrix_func(), transpose_scale_func(), nll_grad_tiles_func()};
    cudaGraphNode_t found[3] = {nullptr, nullptr, nullptr};
    for (size_t i = 0; i < nn; ++i) {
      cudaGraphNodeType ty;
      if (cudaGraphNodeGetType(nodes[i], &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
      cudaKernelNodeParams kpar;
      if (cudaGraphKernelNodeGetParams(nodes[i], &kpar) != cudaSuccess) continue;
      for (int q = 0; q < 3; ++q) if (kpar.func == want[q]) found[q] = nodes[i];
    }
    cudaGetLastError();
    if (!found[0] || (dc > 0 && !found[1]) || !found[2]) { cudaGraphExecDestroy(exec); cudaGraphDestroy(graph); return 1; }
    h->nll_graph = graph; h->nll_exec = exec;
    for (int q = 0; q < 3; ++q) h->nll_nodes[q] = found[q];
    h->nll_key[0] = X; h->nll_key[1] = Z; h->nll_key[2] = y;
    h->nll_key_dims[0] = N; h->nll_key_dims[1] = dc; h->nll_key_dims[2] = dk; h->nll_key_dims[3] = n_valid;
    h->nll_key_dims[4] = n_metrics;
    bufs(h->nll_bufs);
  }
  h->kp = kp; h->sn2 = sn2; h->mean_const = 0.0;
  // new hyper-parameters, by the argument positions pinned in launchers.h (static_asserted against the kernels)
  const int arg_idx[3] = {kKernelMatrixKpArg, kTransposeScaleKpArg, kNllGradTilesKpArg};
  const int arg_cnt[3] = {kKernelMatrixArgs, kTransposeScaleArgs, kNllGradTilesArgs};
  for (int q = 0; q < 3; ++q) {
    if (!h->nll_nodes[q]) continue;
    cudaKernelNodeParams kpar;
    VZ_CUDA(cudaGraphKernelNodeGetParams(h->nll_nodes[q], &kpar));
    void* args[16];
    const int nargs = arg_cnt[q];
    for (int a2 = 0; a2 < nargs; ++a2) args[a2] = kpar.kernelParams[a2];
    args[arg_idx[q]] = &kp;
    if (q == 0) args[kKernelMatrixDiagArg] = &sn2;
    kpar.kernelParams = args;
    VZ_CUDA(cudaGraphExecKernelNodeSetParams(h->nll_exec, h->nll_nodes[q], &kpar));
  }
  VZ_CUDA(cudaGraphLaunch(h->nll_exec, h->stream));
  h->launches += h->nll_launches;
  int bad = 0;
  VZ_CUDA(cudaMemcpyAsync(host2, h->small.as<char>() + kOffLogdet, sizeof(double) * 2, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(hostg, h->small.as<char>() + kOffGrad, sizeof(double) * nq, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(&bad, h->small.as<char>() + kOffFlag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  h->nll_route = VZGP_NLL_GRAPH; h->factor_route = h->nll_factor_route;
  return bad ? 1 : 0;
}

// loss and gradient from the device sums (regularisers: tuned_gp_models.py:167,180,192,269 ->
// 0.01 log(x/c)^2, derivative 0.02 log(x/c) / x).  hostg: [Dk cat | Dc cont | trace | sum G K].
static void finish_loss(const vzgp_params* p, int Dc, int Dk, int n_valid, int n_metrics, double half_logdet_plus_quad,
                        const double* hostg, double* loss_out, double* grad_out, double sum_alpha = 0.0) {
  auto reg = [](double x, double c) { double l = std::log(x / c); return 0.01 * l * l; };
  auto dreg = [](double x, double c) { return 0.02 * std::log(x / c) / x; };
  const double sf2 = p->signal_variance, sn2 = p->observation_noise_variance;
  const bool lin = p->linear_coef != 0.0;
  const int o = Dk + Dc, tail = o + (lin ? 3 : 0);            // position of [noise, signal] in the output
  double loss = half_logdet_plus_quad + 0.5 * n_metrics * n_valid * std::log(2.0 * M_PI);
  loss += reg(sf2, 0.039) + reg(sn2, 0.0039);
  for (int k = 0; k < Dk; ++k) {
    const double l = p->categorical_length_scale_squared[k];
    loss += reg(l, 0.5);
    grad_out[k] = -0.5 * hostg[k] / (l * l) + dreg(l, 0.5);
  }
  const double c = p->linear_coef, s = p->linear_slope_amplitude, lin_a = (c * s) * (c * s);
  for (int d = 0; d < Dc; ++d) {
    const double l = p->continuous_length_scale_squared[d];
    loss += reg(l, 0.5);
    double gd = -0.5 * hostg[Dk + d] / (l * l);
    // K_lin = A sum_d u_id u_jd, u = x w - b, w = l^-1/2:  dK_lin/dl = A (x_i u_j + x_j u_i) (-w^3 / 2)
    if (lin) gd += 0.5 * lin_a * hostg[o + 2 + d] * (-0.5 / (l * std::sqrt(l)));
    grad_out[Dk + d] = gd + dreg(l, 0.5);
  }
  if (lin) {   // tuned_gp_models.py:203-245: slope in the amplitude bounds, shift and mean with 0.5 x^2
    const double q = hostg[o + 2 + Dc], hs = hostg[o + 2 + Dc + 1], h = p->linear_shift, m = p->mean_constant;
    loss += reg(s, 0.039) + 0.5 * h * h + 0.5 * m * m;
    grad_out[o] = 0.5 * (-hs) * lin_a * c + h;                       // d/d shift
    grad_out[o + 1] = 0.5 * q * 2.0 * c * c * s + dreg(s, 0.039);    // d/d slope amplitude
    grad_out[o + 2] = -c * sum_alpha + m;                            // d/d mean constant
  }
  grad_out[tail] = 0.5 * hostg[o] + dreg(sn2, 0.0039);
  grad_out[tail + 1] = 0.5 * hostg[o + 1] / sf2 + dreg(sf2, 0.039);
  *loss_out = loss;
}

// ---------------------------------------------------------------------------
// R evaluations (the ARD restarts, one handle each) as ONE graph launch: the R launch sequences are captured
// as parallel branches (fork / join by events on the handles' streams), each ending with the copies of its
// results into that handle's pinned host block.  One cudaGraphLaunch + one synchronisation per round of the
// lock-step L-BFGS-B driver (ard.py) instead of R host threads contending for the driver lock.
// ---------------------------------------------------------------------------
constexpr int kMaxBatch = 16;
struct BatchGraph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  cudaGraphNode_t nodes[kMaxBatch][3] = {};
  cudaEvent_t fork = nullptr, join[kMaxBatch] = {};
  const void* key_ptr[3] = {nullptr, nullptr, nullptr};
  int key_dims[6] = {0, 0, 0, 0, 0, 0};          // N, dc, dk, n_valid, n_metrics, R
  const vzgp_handle* hs[kMaxBatch] = {};
  const void* bufs[kMaxBatch][kNllBufs] = {};
  int launches = 0;
};

static void batch_drop(BatchGraph* b) {
  if (b->exec) cudaGraphExecDestroy(b->exec);
  if (b->graph) cudaGraphDestroy(b->graph);
  b->exec = nullptr; b->graph = nullptr;
}

static void handle_bufs(vzgp_handle* h, const void** o) {
  const DevBuf* b[kNllBufs] = {&h->X, &h->XT, &h->Z, &h->L, &h->Linv, &h->alpha, &h->ypad, &h->Kws, &h->Tws, &h->Kinv, &h->small,
                               &h->LinvT, &h->df_tasks[1], &h->df_flags, &h->df_S};
  for (int q = 0; q < kNllBufs; ++q) o[q] = b[q]->ptr;
}

static int ensure_pinned(vzgp_handle* h, size_t bytes) {
  if (h->pinned && h->pinned_bytes >= bytes) return 0;
  if (h->pinned) cudaFreeHost(h->pinned);
  h->pinned = nullptr; h->pinned_bytes = 0;
  VZ_CUDA(cudaMallocHost(&h->pinned, bytes));
  h->pinned_bytes = bytes;
  return 0;
}

// The acquisition function the scoring calls on h evaluate (nullptr: UCB with the call's coefficient).
static const AcqFn* handle_acq(const vzgp_handle* h) { return h->has_acq_fn ? &h->acq_fn : nullptr; }

static int acq_term_from(const vzgp_acq_term& t, AcqTerm* out) {
  VZ_ARG(t.kind >= VZGP_ACQ_UCB && t.kind <= VZGP_ACQ_PI, "unknown vzgp_acq_kind");
  VZ_ARG(std::isfinite(t.coefficient) || t.kind == VZGP_ACQ_EI || t.kind == VZGP_ACQ_PI, "finite coefficient");
  VZ_ARG((t.kind != VZGP_ACQ_EI && t.kind != VZGP_ACQ_PI) || (std::isfinite(t.best_label) && std::isfinite(t.exploration)),
         "EI / PI need a finite best_label and exploration");
  out->kind = t.kind; out->coefficient = t.coefficient; out->best_label = t.best_label; out->exploration = t.exploration;
  return 0;
}

}  // namespace vzgp

using namespace vzgp;

extern "C" {

const char* vzgp_last_error(void) { return g_err; }
int vzgp_version(void) { return 3; }

int vzgp_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int vzgp_create(int device, void* stream, vzgp_handle** out) {
  VZ_ARG(out != nullptr, "out");
  *out = nullptr;
  int n = 0;
  VZ_CUDA(cudaGetDeviceCount(&n));
  VZ_ARG(device >= 0 && device < n, "device ordinal");
  Guard g(device);
  vzgp_handle* h = new vzgp_handle();
  h->device = device;
  if (stream) {
    h->stream = reinterpret_cast<cudaStream_t>(stream);
  } else {
    cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
      set_error("cudaStreamCreate: %s", cudaGetErrorString(e));
      delete h;
      return VZGP_ERR_CUDA;
    }
    h->own_stream = true;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->sm_count = prop.multiProcessorCount;
  int s = h->small.reserve(kSmallBytes);
  if (s < 0) { delete h; return s; }
  cudaMemsetAsync(h->small.ptr, 0, kSmallBytes, h->stream);
  *out = h;
  return 0;
}

static void eagle_step_free(vzgp_handle* h);

int vzgp_destroy(vzgp_handle* h) {
  if (!h) return 0;
  Guard g(h->device);
  cudaStreamSynchronize(h->stream);
  for (DevBuf* b : {&h->X, &h->Z, &h->L, &h->Linv, &h->alpha, &h->ypad, &h->Kws, &h->Tws, &h->Kinv, &h->XT,
                    &h->scratch, &h->small, &h->xs_dev, &h->out_dev, &h->eagle, &h->pe_tmp, &h->pe_multi_tmp,
                    &h->LinvT, &h->df_tasks[0], &h->df_tasks[1], &h->df_flags, &h->df_S, &h->scal, &h->gen,
                    &h->i8_planes, &h->i8_scale, &h->i8_kdig})
    b->release();
  eagle_step_free(h);
  if (h->pinned) cudaFreeHost(h->pinned);
  if (h->copy_stream) {
    for (int i = 0; i < 4; ++i) cudaEventDestroy(h->copy_ev[i]);
    cudaStreamDestroy(h->copy_stream);
  }
  if (h->nll_exec) cudaGraphExecDestroy(h->nll_exec);
  if (h->nll_graph) cudaGraphDestroy(h->nll_graph);
  if (h->batch) {
    BatchGraph* b = static_cast<BatchGraph*>(h->batch);
    batch_drop(b);
    if (b->fork) { cudaEventDestroy(b->fork); for (int r = 0; r < kMaxBatch; ++r) cudaEventDestroy(b->join[r]); }
    delete b;
  }
  if (h->own_stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int vzgp_synchronize(vzgp_handle* h) {
  VZ_ARG(h != nullptr, "handle");
  Guard g(h->device);
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

int64_t vzgp_launch_count(const vzgp_handle* h) { return h ? h->launches : 0; }

int vzgp_set_int(vzgp_handle* h, const char* key, int value) {
  VZ_ARG(h && key, "handle / key");
  if (std::strcmp(key, "dataflow_ctas") == 0) { VZ_ARG(value >= 0, "value >= 0"); h->df_ctas = value; return 0; }
  if (std::strcmp(key, "score_i8") == 0) { VZ_ARG(value >= -1 && value <= 1, "value in {-1, 0, 1}"); h->score_i8 = value; return 0; }
  if (std::strcmp(key, "small_tiles") == 0) { VZ_ARG(value >= -1, "value >= -1"); h->small_tiles = value; return 0; }
  set_error("vzgp_set_int: unknown key '%s'", key);
  return VZGP_ERR_ARG;
}

int vzgp_set_acquisition(vzgp_handle* h, const vzgp_acq_fn* fn) {
  VZ_ARG(h != nullptr, "handle");
  if (fn == nullptr) { h->has_acq_fn = false; return 0; }
  AcqFn f = ucb_acq_fn(0.0);
  VZ_TRY(acq_term_from(fn->main, &f.main));
  f.use_thr = fn->use_threshold ? 1 : 0;
  if (f.use_thr) {
    VZ_TRY(acq_term_from(fn->thresholding, &f.thr));
    VZ_ARG(!std::isnan(fn->threshold), "threshold is NaN (pass use_threshold = 0)");
    VZ_ARG(std::isfinite(fn->bad_acq_value), "finite bad_acq_value");
    f.threshold = fn->threshold;
    f.bad_value = fn->bad_acq_value;
  }
  h->acq_fn = f;
  h->has_acq_fn = true;
  return 0;
}

int vzgp_get_int(const vzgp_handle* h, const char* key, int64_t* value) {
  VZ_ARG(h && key && value, "handle / key / value");
  if (std::strcmp(key, "launches") == 0) { *value = h->launches; return 0; }
  if (std::strcmp(key, "score_i8_launches") == 0) { *value = h->i8_launches; return 0; }
  if (std::strcmp(key, "sm_count") == 0) { *value = h->sm_count; return 0; }
  if (std::strcmp(key, "score_route") == 0) { *value = h->score_route; return 0; }
  if (std::strcmp(key, "score_nsplit") == 0) { *value = h->score_nsplit; return 0; }
  if (std::strcmp(key, "score_grid") == 0) { *value = h->score_grid; return 0; }
  if (std::strcmp(key, "nll_route") == 0) { *value = h->nll_route; return 0; }
  if (std::strcmp(key, "factor_route") == 0) { *value = h->factor_route; return 0; }
  set_error("vzgp_get_int: unknown key '%s'", key);
  return VZGP_ERR_ARG;
}

int vzgp_kernel_matrix(vzgp_handle* h, const double* X, const int32_t* Z, int N, int Dc, int Dk,
                       int n_valid, const vzgp_params* p, double diag_add, double* K, int ldk) {
  VZ_ARG(h && K, "handle / K");
  VZ_ARG(N >= 1 && ldk >= N, "N, ldk");
  VZ_ARG(n_valid >= 0 && n_valid <= N, "n_valid");
  Guard g(h->device);
  KernelParams kp;
  VZ_TRY(fill_kernel_params(p, Dc, Dk, &kp));
  return launch_kernel_matrix(h, X, Z, N, n_valid, kp, diag_add, K, ldk);
}

int vzgp_cross_kernel(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const double* X,
                      const int32_t* Z, int N, int Dc, int Dk, const vzgp_params* p, double* Ks,
                      int ldks) {
  VZ_ARG(h && Ks, "handle / Ks");
  VZ_ARG(M >= 1 && N >= 1 && ldks >= N, "M, N, ldks");
  Guard g(h->device);
  KernelParams kp;
  VZ_TRY(fill_kernel_params(p, Dc, Dk, &kp));
  return launch_cross_kernel(h, Xs, Zs, M, X, Z, N, N, kp, Ks, ldks);
}

// Copies the top-left [N x N] lower part of a padded [np x np] matrix into a user matrix.
__global__ void k_unpad_lower(const double* __restrict__ src, int np, int N, double* __restrict__ dst,
                              int ld) {
  int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j < N) dst[(size_t)i * ld + j] = (j <= i) ? src[(size_t)i * np + j] : 0.0;
}

int vzgp_cholesky_retry(vzgp_handle* h, const double* A, int N, int lda, double jitter0,
                        int max_iters, double* L, int ldl, double* shift_out) {
  VZ_ARG(h && A && L, "handle / A / L");
  VZ_ARG(N >= 1 && lda >= N && ldl >= N, "N, lda, ldl");
  VZ_ARG(max_iters >= 0, "max_iters");
  Guard g(h->device);
  const int np = round_up(N, kBlk);
  VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * 2));
  double* Lp = h->Kinv.as<double>();
  double* Li = Lp + (size_t)np * np;
  int retries = cholesky_retry_padded(h, A, lda, N, np, jitter0, max_iters, Lp, Li, shift_out);
  if (retries < 0) return retries;
  k_unpad_lower<<<dim3((N + 255) / 256, N), 256, 0, h->stream>>>(Lp, np, N, L, ldl);
  VZ_CHECK_LAUNCH();
  h->launches++;
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  return retries;
}

int vzgp_factor_inverse(vzgp_handle* h, const double* A, int N, int lda, double* L, double* Linv, double* Kinv,
                        int ld) {
  VZ_ARG(h && A && L && Linv, "handle / A / L / Linv");
  VZ_ARG(N >= 1 && lda >= N && ld >= N, "N, lda, ld");
  Guard g(h->device);
  const int np = round_up(N, kBlk);
  VZ_TRY(ensure_model_buffers(h, np, 1, 0));
  h->fitted = false; h->i8_ready = false;
  const bool want_kinv = Kinv != nullptr;
  if (want_kinv) VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * kLauumSplit));
  int* flag = reinterpret_cast<int*>(h->small.as<char>() + kOffFlag);
  VZ_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), h->stream));
  VZ_CUDA(cudaMemsetAsync(h->Linv.as<double>(), 0, sizeof(double) * (size_t)np * np, h->stream));
  VZ_TRY(launch_copy_lower_shift(h, A, lda, N, np, 0.0, h->L.as<double>(), np));
  bool df = false;
  VZ_TRY(factor_invert(h, h->L.as<double>(), h->Linv.as<double>(), h->LinvT.as<double>(),
                       want_kinv ? h->Kinv.as<double>() : nullptr, np, flag, &df));
  if (want_kinv && !df) {
    // panel-kernel fallback: K^-1 as kLauumSplit partial planes; sum them into plane 0's lower triangle
    VZ_TRY(launch_lauum(h, h->Linv.as<double>(), np, h->Kinv.as<double>(), np, np));
    VZ_TRY(launch_sum_planes(h, h->Kinv.as<double>(), np, lauum_plane_rows(np)));
  }
  k_unpad_lower<<<dim3((N + 255) / 256, N), 256, 0, h->stream>>>(h->L.as<double>(), np, N, L, ld);
  k_unpad_lower<<<dim3((N + 255) / 256, N), 256, 0, h->stream>>>(h->Linv.as<double>(), np, N, Linv, ld);
  if (want_kinv) k_unpad_lower<<<dim3((N + 255) / 256, N), 256, 0, h->stream>>>(h->Kinv.as<double>(), np, N, Kinv, ld);
  VZ_CHECK_LAUNCH();
  h->launches += want_kinv ? 3 : 2;
  int bad = 0, to = 0;
  VZ_CUDA(cudaMemcpyAsync(&bad, flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  if (df) {
    VZ_TRY(chol_dataflow_timed_out(h, &to));
    if (to) { set_error("dataflow factorisation: a tile wait timed out"); return VZGP_ERR_CUDA; }
  }
  return bad ? 1 : 0;
}

int vzgp_tri_inverse(vzgp_handle* h, const double* L, int N, int ldl, double* Linv, int ldi) {
  VZ_ARG(h && L && Linv, "handle / L / Linv");
  VZ_ARG(N >= 1 && ldl >= N && ldi >= N, "N, ldl, ldi");
  Guard g(h->device);
  const int np = round_up(N, kBlk);
  VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * 3));
  double* Lp = h->Kinv.as<double>();
  double* Li = Lp + (size_t)np * np;
  double* T = Li + (size_t)np * np;
  VZ_TRY(launch_copy_lower_shift(h, L, ldl, N, np, 0.0, Lp, np));
  VZ_CUDA(cudaMemsetAsync(Li, 0, sizeof(double) * (size_t)np * np, h->stream));
  VZ_TRY(launch_diag_inv(h, Lp, np, Li, np, np));
  VZ_TRY(trtri_doubling(h, Lp, np, Li, np, T, np, np));
  k_unpad_lower<<<dim3((N + 255) / 256, N), 256, 0, h->stream>>>(Li, np, N, Linv, ldi);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int vzgp_fit_multi(vzgp_handle* h, const double* X, const int32_t* Z, const double* Y, int N, int Dc,
                   int Dk, int n_valid, int n_metrics, const vzgp_params* p) {
  VZ_ARG(h != nullptr, "handle");
  Guard g(h->device);
  int retries = fit_common(h, X, Z, Y, N, Dc, Dk, n_valid, p, nullptr, n_metrics);
  if (retries < 0) return retries;
  h->fitted = true;
  return retries;
}

int vzgp_fit(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int Dc,
             int Dk, int n_valid, const vzgp_params* p) {
  return vzgp_fit_multi(h, X, Z, y, N, Dc, Dk, n_valid, 1, p);
}

int vzgp_get_cholesky(vzgp_handle* h, double* L, int ldl) {
  VZ_ARG(h && L, "handle / L");
  if (!h->fitted) { set_error("vzgp_get_cholesky: model not fitted"); return VZGP_ERR_STATE; }
  VZ_ARG(ldl >= h->n, "ldl");
  Guard g(h->device);
  k_unpad_lower<<<dim3((h->n + 255) / 256, h->n), 256, 0, h->stream>>>(h->L.as<double>(), h->np, h->n, L, ldl);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

int vzgp_get_alpha(vzgp_handle* h, double* alpha) {
  VZ_ARG(h && alpha, "handle / alpha");
  if (!h->fitted) { set_error("vzgp_get_alpha: model not fitted"); return VZGP_ERR_STATE; }
  Guard g(h->device);
  VZ_CUDA(cudaMemcpyAsync(alpha, h->alpha.ptr, sizeof(double) * h->n, cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

int vzgp_nll_grad(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int Dc,
                  int Dk, int n_valid, const vzgp_params* p, double* loss_out, double* grad_out) {
  return vzgp_nll_grad_multi(h, X, Z, y, N, Dc, Dk, n_valid, 1, p, loss_out, grad_out);
}

int vzgp_nll_grad_multi(vzgp_handle* h, const double* X, const int32_t* Z, const double* y, int N, int Dc,
                        int Dk, int n_valid, int n_metrics, const vzgp_params* p, double* loss_out, double* grad_out) {
  VZ_ARG(h && loss_out && grad_out, "handle / outputs");
  VZ_ARG(n_metrics >= 1 && n_metrics <= kMaxMetrics, "1 <= n_metrics <= 8");
  Guard g(h->device);
  auto finish = [&](double half_logdet_plus_quad, const double* hostg) {
    finish_loss(p, Dc, Dk, n_valid, n_metrics, half_logdet_plus_quad, hostg, loss_out, grad_out);
  };
  static const bool small_ok = [] { const char* e = getenv("VZGP_NLL_SMALL"); return !(e && e[0] == '0'); }();
  const bool lin = p->linear_coef != 0.0;
  VZ_ARG(!lin || n_metrics == 1, "linear_coef with several metrics is not implemented");
  if (N <= kBlk && small_ok && n_metrics == 1 && !lin) {
    // Small studies: the whole evaluation is one single-CTA kernel (nll_small.cu).  The handle's
    // fitted model is not touched (ARD callers refit with the chosen parameters afterwards).
    VZ_ARG(N >= 1 && n_valid >= 1 && n_valid <= N, "1 <= n_valid <= N");
    VZ_ARG(X != nullptr || Dc == 0, "X");
    VZ_ARG(Z != nullptr || Dk == 0, "Z");
    VZ_ARG(y != nullptr, "y");
    KernelParams kp;
    VZ_TRY(fill_kernel_params(p, Dc, Dk, &kp));
    const int nq = Dc + Dk + 2;
    double* dout = reinterpret_cast<double*>(h->small.as<char>() + kOffGrad);   // 4 + nq doubles
    VZ_TRY(launch_nll_grad_small(h, X, Z, y, N, n_valid, kp, p->observation_noise_variance, 1e-4, 5, dout));
    double host[4 + kMaxGrad];
    VZ_CUDA(cudaMemcpyAsync(host, dout, sizeof(double) * (4 + nq), cudaMemcpyDeviceToHost, h->stream));
    VZ_CUDA(cudaStreamSynchronize(h->stream));
    h->nll_route = VZGP_NLL_SMALL; h->factor_route = VZGP_FACTOR_PANEL;
    finish(host[0] + host[1], host + 4);
    return (int)host[3];
  }
  if (!lin) {
    // Replayed graph (no retry inside); a flagged pivot or any graph problem falls through to the
    // eager path below, which has the jitter loop.
    VZ_ARG(N >= 1 && n_valid >= 1 && n_valid <= N, "1 <= n_valid <= N");
    VZ_ARG(X != nullptr || Dc == 0, "X");
    VZ_ARG(Z != nullptr || Dk == 0, "Z");
    VZ_ARG(y != nullptr, "y");
    double g2[2], gg[kMaxGrad];
    const int st = nll_graph_eval(h, X, Z, y, N, Dc, Dk, n_valid, n_metrics, p, g2, gg);
    if (st < 0) return st;
    if (st == 0) {
      finish(g2[1] + g2[0], gg);
      return 0;
    }
  }
  double shift = 0.0;
  int retries = fit_common(h, X, Z, y, N, Dc, Dk, n_valid, p, &shift, n_metrics);
  if (retries < 0) return retries;
  h->nll_route = VZGP_NLL_EAGER;
  const int np = h->np, nq = Dc + Dk + 2 + (lin ? Dc + 2 : 0);
  VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * kLauumSplit));   // partial planes of K_y^-1
  double* out2 = reinterpret_cast<double*>(h->small.as<char>() + kOffLogdet);
  double* gout = reinterpret_cast<double*>(h->small.as<char>() + kOffGrad);
  double* w = h->ypad.as<double>() + np;
  VZ_TRY(launch_logdet_quad(h, h->L.as<double>(), np, N, n_valid, w, out2, 4 * np, n_metrics, h->alpha.as<double>()));
  VZ_TRY(launch_lauum(h, h->Linv.as<double>(), np, h->Kinv.as<double>(), np, np));
  VZ_TRY(launch_nll_grad_tiles(h, h->X.as<double>(), h->Z.as<int32_t>(), np, n_valid, h->kp,
                               h->Kinv.as<double>(), np, h->alpha.as<double>(), h->Tws.as<double>(), gout, 0, n_metrics));
  double host2[3];
  double hostg[kMaxGrad];
  VZ_CUDA(cudaMemcpyAsync(host2, out2, sizeof(host2), cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(hostg, gout, sizeof(double) * nq, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  finish_loss(p, Dc, Dk, n_valid, n_metrics, host2[1] + host2[0], hostg, loss_out, grad_out, host2[2]);
  return retries;
}

static int check_scoring(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M,
                         const vzgp_acq* acq, const double* score) {
  VZ_ARG(h != nullptr, "handle");
  if (!h->fitted) { set_error("scoring requested before vzgp_fit"); return VZGP_ERR_STATE; }
  VZ_ARG(M >= 0, "M");
  VZ_ARG(acq != nullptr, "acq");
  VZ_ARG(score != nullptr, "score");
  VZ_ARG(Xs != nullptr || h->dc == 0, "Xs");
  VZ_ARG(Zs != nullptr || h->dk == 0, "Zs");
  return 0;
}

int vzgp_score(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
               double* score, double* mu, double* sigma, double* linf) {
  if (h != nullptr && h->fitted && M == 0) return 0;  // empty pool: nothing to do
  VZ_TRY(check_scoring(h, Xs, Zs, M, acq, score));
  Guard g(h->device);
  return launch_score(h, Xs, Zs, M, acq, score, mu, sigma, linf, handle_acq(h));
}

int vzgp_clamped_count(vzgp_handle* h, int64_t* count_out) {
  VZ_ARG(h && count_out, "handle / out");
  Guard g(h->device);
  int c = 0;
  int* d = reinterpret_cast<int*>(h->small.as<char>() + kOffClamp);
  VZ_CUDA(cudaMemcpyAsync(&c, d, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemsetAsync(d, 0, sizeof(int), h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  *count_out = c;
  return 0;
}

// Host candidates -> device staging -> scores in h->out_dev[0..M) (+ mu / sigma / linf planes), all
// enqueued on the handle's stream, nothing copied back, no synchronisation.  The host->device copy is
// pipelined against the scoring: candidates go over in up to three chunks sized in whole waves of
// 64-row tiles (1 wave, 3 waves, rest) on a copy stream, and the score launch of chunk c only waits for
// the event of chunk c.
static int score_host_enqueue(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                              bool mu, bool sigma, bool linf, double** dX_out, double** o_out) {
  const size_t xb = sizeof(double) * (size_t)M * h->dc, zb = sizeof(int32_t) * (size_t)M * h->dk;
  VZ_TRY(h->xs_dev.reserve(xb + zb + 64));
  VZ_TRY(h->out_dev.reserve(sizeof(double) * (size_t)M * 4));
  double* dX = h->xs_dev.as<double>();
  int32_t* dZ = reinterpret_cast<int32_t*>(h->xs_dev.as<char>() + ((xb + 15) / 16) * 16);
  double* o = h->out_dev.as<double>();
  if (!h->copy_stream) {
    VZ_CUDA(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i) VZ_CUDA(cudaEventCreateWithFlags(&h->copy_ev[i], cudaEventDisableTiming));
  }
  const int wave = h->sm_count * 64;
  int bounds[4] = {0, 0, 0, 0};
  int nchunk = 0;
  {
    int pos = 0;
    // one wave, three waves, the rest: every copy lands while the previous chunk is being scored
    const int plan[2] = {wave, 3 * wave};
    for (int i = 0; i < 2 && M - pos > 2 * plan[i]; ++i) { pos += plan[i]; bounds[++nchunk] = pos; }
    bounds[++nchunk] = M;
  }
  VZ_CUDA(cudaEventRecord(h->copy_ev[3], h->stream));          // previous users of the staging buffers
  VZ_CUDA(cudaStreamWaitEvent(h->copy_stream, h->copy_ev[3], 0));
  for (int c = 0; c < nchunk; ++c) {
    const size_t lo = bounds[c], n = bounds[c + 1] - bounds[c];
    if (h->dc > 0) VZ_CUDA(cudaMemcpyAsync(dX + lo * h->dc, Xs + lo * h->dc, sizeof(double) * n * h->dc, cudaMemcpyHostToDevice, h->copy_stream));
    if (h->dk > 0) VZ_CUDA(cudaMemcpyAsync(dZ + lo * h->dk, Zs + lo * h->dk, sizeof(int32_t) * n * h->dk, cudaMemcpyHostToDevice, h->copy_stream));
    VZ_CUDA(cudaEventRecord(h->copy_ev[c], h->copy_stream));
  }
  for (int c = 0; c < nchunk; ++c) {
    const size_t lo = bounds[c];
    const int n = bounds[c + 1] - bounds[c];
    VZ_CUDA(cudaStreamWaitEvent(h->stream, h->copy_ev[c], 0));
    VZ_TRY(launch_score(h, dX + lo * h->dc, h->dk > 0 ? dZ + lo * h->dk : nullptr, n, acq, o + lo, mu ? o + M + lo : nullptr,
                        sigma ? o + 2 * (size_t)M + lo : nullptr, linf ? o + 3 * (size_t)M + lo : nullptr, handle_acq(h)));
  }
  *dX_out = dX;
  *o_out = o;
  return 0;
}

int vzgp_score_host(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M,
                    const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf) {
  VZ_TRY(check_scoring(h, Xs, Zs, M, acq, score));
  if (M == 0) return 0;
  Guard g(h->device);
  double *dX, *o;
  VZ_TRY(score_host_enqueue(h, Xs, Zs, M, acq, mu != nullptr, sigma != nullptr, linf != nullptr, &dX, &o));
  const size_t ob = sizeof(double) * (size_t)M;
  VZ_CUDA(cudaMemcpyAsync(score, o, ob, cudaMemcpyDeviceToHost, h->stream));
  if (mu) VZ_CUDA(cudaMemcpyAsync(mu, o + M, ob, cudaMemcpyDeviceToHost, h->stream));
  if (sigma) VZ_CUDA(cudaMemcpyAsync(sigma, o + 2 * (size_t)M, ob, cudaMemcpyDeviceToHost, h->stream));
  if (linf) VZ_CUDA(cudaMemcpyAsync(linf, o + 3 * (size_t)M, ob, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

static int topk_to_device(vzgp_handle* h, const double* score, int64_t M, int count,
                          long long** d_idx, double** d_val) {
  VZ_ARG(count >= 1 && count <= kMaxTopk, "1 <= count <= 256");
  *d_idx = reinterpret_cast<long long*>(h->small.as<char>() + kOffTopIdx);
  *d_val = reinterpret_cast<double*>(h->small.as<char>() + kOffTopVal);
  ArgMax* part = reinterpret_cast<ArgMax*>(h->small.as<char>() + kOffPartial);
  int64_t nb = (M + 2047) / 2048;
  if (nb < 1) nb = 1;
  if (nb > 2048) nb = 2048;
  return launch_topk_device(h, score, M, count, *d_idx, *d_val, part, (int)nb);
}

int vzgp_topk(vzgp_handle* h, const double* score, int64_t M, int count, int64_t* idx_out,
              double* val_out) {
  VZ_ARG(h && score && idx_out && val_out, "handle / pointers");
  VZ_ARG(M >= 1, "M");
  Guard g(h->device);
  long long* d_idx; double* d_val;
  VZ_TRY(topk_to_device(h, score, M, count, &d_idx, &d_val));
  long long hidx[kMaxTopk];
  VZ_CUDA(cudaMemcpyAsync(hidx, d_idx, sizeof(long long) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(val_out, d_val, sizeof(double) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  for (int c = 0; c < count; ++c) idx_out[c] = (hidx[c] == LLONG_MAX) ? -1 : (int64_t)hidx[c];
  return 0;
}

int vzgp_random_pool(vzgp_handle* h, int64_t M, int Dc, int64_t index_base, uint64_t seed, double* X) {
  VZ_ARG(h && X, "handle / X");
  VZ_ARG(M >= 0 && Dc >= 1, "M, Dc");
  Guard g(h->device);
  return launch_random_fill(h, X, M * Dc, index_base * Dc, seed, 3u, 0u);
}

static int check_cat_sizes(const vzgp_handle* h, const int32_t* cat_sizes, int* sizes, int* smax) {
  *smax = 0;
  for (int k = 0; k < kMaxDk; ++k) sizes[k] = 1;
  if (h->dk == 0) return 0;
  VZ_ARG(cat_sizes != nullptr, "cat_sizes is required when the model has categorical features");
  for (int k = 0; k < h->dk; ++k) {
    VZ_ARG(cat_sizes[k] >= 1 && cat_sizes[k] <= 64, "1 <= cat_sizes[k] <= 64");
    sizes[k] = cat_sizes[k];
    if (sizes[k] > *smax) *smax = sizes[k];
  }
  return 0;
}

int vzgp_random_pool_cat(vzgp_handle* h, int64_t M, int Dk, const int32_t* cat_sizes, int64_t index_base,
                         uint64_t seed, int32_t* Z) {
  VZ_ARG(h && Z && cat_sizes, "handle / Z / cat_sizes");
  VZ_ARG(M >= 0 && Dk >= 1 && Dk <= kMaxDk, "M, Dk");
  Guard g(h->device);
  int sizes[kMaxDk];
  for (int k = 0; k < Dk; ++k) {
    VZ_ARG(cat_sizes[k] >= 1, "cat_sizes[k] >= 1");
    sizes[k] = cat_sizes[k];
  }
  return launch_random_fill_cat(h, Z, M, Dk, sizes, index_base, seed, 8u);
}

int vzgp_random_search(vzgp_handle* h, int64_t M, int64_t index_base, const vzgp_acq* acq,
                       const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                       double* best_score, int64_t* best_index) {
  VZ_ARG(h && acq && best_score, "handle / pointers");
  if (!h->fitted) { set_error("vzgp_random_search before vzgp_fit"); return VZGP_ERR_STATE; }
  VZ_ARG(M >= 1 && M <= INT_MAX, "1 <= M < 2^31 per call");
  VZ_ARG(best_x != nullptr || h->dc == 0, "best_x");
  VZ_ARG(best_z != nullptr || h->dk == 0, "best_z");
  Guard g(h->device);
  const int dc = h->dc, dk = h->dk;
  int sizes[kMaxDk], smax;
  VZ_TRY(check_cat_sizes(h, cat_sizes, sizes, &smax));
  const size_t xb = sizeof(double) * (size_t)M * (dc > 0 ? dc : 1);
  VZ_TRY(h->xs_dev.reserve(xb + sizeof(int32_t) * (size_t)M * (dk > 0 ? dk : 1) + 64));
  VZ_TRY(h->out_dev.reserve(sizeof(double) * ((size_t)M + (size_t)kMaxTopk * (dc + dk + 1))));
  double* dX = h->xs_dev.as<double>();
  int32_t* dZ = reinterpret_cast<int32_t*>(h->xs_dev.as<char>() + ((xb + 15) / 16) * 16);
  double* dS = h->out_dev.as<double>();
  double* dBest = dS + M;
  int32_t* dBestZ = reinterpret_cast<int32_t*>(dBest + (size_t)kMaxTopk * (dc > 0 ? dc : 1));
  if (dc > 0) VZ_TRY(launch_random_fill(h, dX, M * dc, index_base * dc, seed, 3u, 0u));
  if (dk > 0) VZ_TRY(launch_random_fill_cat(h, dZ, M, dk, sizes, index_base, seed, 8u));
  VZ_TRY(launch_score(h, dX, dk > 0 ? dZ : nullptr, (int)M, acq, dS, nullptr, nullptr, nullptr, handle_acq(h)));
  long long* d_idx; double* d_val;
  VZ_TRY(topk_to_device(h, dS, M, count, &d_idx, &d_val));
  if (dc > 0) VZ_TRY(launch_gather_rows(h, dX, dc, d_idx, count, M, dBest));
  if (dk > 0) VZ_TRY(launch_gather_rows_i32(h, dZ, dk, d_idx, count, M, dBestZ));
  long long hidx[kMaxTopk];
  VZ_CUDA(cudaMemcpyAsync(hidx, d_idx, sizeof(long long) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(best_score, d_val, sizeof(double) * count, cudaMemcpyDeviceToHost, h->stream));
  if (dc > 0) VZ_CUDA(cudaMemcpyAsync(best_x, dBest, sizeof(double) * (size_t)count * dc, cudaMemcpyDeviceToHost, h->stream));
  if (dk > 0) VZ_CUDA(cudaMemcpyAsync(best_z, dBestZ, sizeof(int32_t) * (size_t)count * dk, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  if (best_index)
    for (int c = 0; c < count; ++c)
      best_index[c] = (hidx[c] == LLONG_MAX) ? -1 : (int64_t)hidx[c] + index_base;
  return 0;
}

// Carves handle->eagle into the device-resident optimiser state for (cfg, count) on `h`.
struct EagleScratch {
  double* prior_r;    // [max(n_prior, 1)] rewards of the prior trials
  double* chosen_r;   // [P]
  int* ord;           // [max(n_prior, 1)]
};
static int eagle_setup(vzgp_handle* h, const vzgp_eagle_config* cfg, const int32_t* cat_sizes, int count, uint64_t seed,
                       int n_prior, EagleDev* pe_, EagleScratch* sc) {
  EagleDev& e = *pe_;
  const int q = cfg->n_parallel > 1 ? cfg->n_parallel : 1;
  VZ_ARG(q == 1 || (h->dk == 0 && h->dc * q <= kMaxDc), "n_parallel > 1 needs continuous features only and n_parallel * Dc <= 64");
  const int P = cfg->pool_size, B = cfg->batch_size, D = h->dc * q, Dk = h->dk;
  VZ_TRY(check_cat_sizes(h, cat_sizes, e.sizes, &e.smax));
  e.q = q;
  e.norm_dim = h->dc + h->dk;
  // carve the eagle buffer: doubles | long longs | ints
  const size_t np1 = (size_t)(n_prior > 0 ? n_prior : 1);
  const size_t nd = (size_t)P * D + 2 * (size_t)P + 8 + (size_t)B * D + B + 2 * ((size_t)count * D + count) + np1 + P;
  const size_t nl = 2 * (size_t)count;
  const size_t ni = 16 + np1 + (size_t)P * Dk + (size_t)B * Dk + 2 * (size_t)count * Dk;
  VZ_TRY(h->eagle.reserve(nd * sizeof(double) + nl * sizeof(long long) + ni * sizeof(int32_t) + 64));
  double* p = h->eagle.as<double>();
  e.pool = p; p += (size_t)P * D;
  e.rewards = p; p += P;
  e.pert = p; p += P;
  e.best_reward = p; p += 8;
  e.batch = p; p += (size_t)B * D;
  e.batch_r = p; p += B;
  e.best_x = p; p += (size_t)count * D;
  e.best_r = p; p += count;
  e.tmp_x = p; p += (size_t)count * D;
  e.tmp_r = p; p += count;
  sc->prior_r = p; p += np1;
  sc->chosen_r = p; p += P;
  long long* lp = reinterpret_cast<long long*>(p);
  e.best_id = lp; lp += count;
  e.tmp_id = lp; lp += count;
  int32_t* ip = reinterpret_cast<int32_t*>(lp);
  e.iter = ip; ip += 16;
  sc->ord = ip; ip += np1;
  e.pool_z = ip; ip += (size_t)P * Dk;
  e.batch_z = ip; ip += (size_t)B * Dk;
  e.best_z = ip; ip += (size_t)count * Dk;
  e.tmp_z = ip; ip += (size_t)count * Dk;
  e.P = P; e.B = B; e.D = D; e.Dk = Dk; e.count = count; e.cfg = *cfg; e.seed = seed;
  return eagle_prepare(e);
}
static int eagle_check_config(const vzgp_handle* h, const vzgp_eagle_config* cfg, int count) {
  VZ_ARG(cfg->pool_size >= 1 && cfg->batch_size >= 1, "pool/batch size");
  VZ_ARG(cfg->pool_size % cfg->batch_size == 0, "pool_size must be a multiple of batch_size");
  VZ_ARG(cfg->pool_size <= 3000, "pool_size <= 3000");
  VZ_ARG(cfg->batch_size <= 8192, "batch_size <= 8192");
  VZ_ARG(count >= 1 && count <= kMaxTopk, "count");
  VZ_ARG(cfg->max_evaluations >= 1, "max_evaluations");
  (void)h;
  return 0;
}

static int eagle_run_impl(vzgp_handle* h, vzgp_handle* hB, const vzgp_eagle_config* cfg, const vzgp_acq* acq,
                          const vzgp_pe_params* pe, const double* prior, const int32_t* prior_z, int n_prior,
                          const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                          double* best_score, vzgp_handle* const* ens = nullptr, int n_ens = 0,
                          const vzgp_scalarization* scal = nullptr, const double* stack_alphas = nullptr,
                          const vzgp_pe_multi_params* pem = nullptr) {
  VZ_ARG(h && cfg && (acq || pe || scal || pem) && best_score, "handle / pointers");
  const AcqFn* fn = (pe || scal || pem) ? nullptr : handle_acq(ens ? ens[0] : h);   // multi-handle calls: the setting of hs[0]
  auto score_batch = [&](const double* xs, const int32_t* zs, int m, double* out) -> int {
    if (pem) return launch_score_pe_multi(h, hB, xs, zs, m, pem, out, nullptr, nullptr, nullptr);
    if (scal) return launch_score_multi(h, xs, zs, m, out, nullptr, nullptr);
    if (pe) return launch_score_pe(h, hB, xs, zs, m, pe, out, nullptr, nullptr, nullptr);
    if (stack_alphas) return launch_score_stack(ens, n_ens, stack_alphas, xs, zs, m, acq, out, nullptr, nullptr, nullptr, fn);
    if (n_ens > 1) return launch_score_ensemble(ens, n_ens, xs, zs, m, acq, out, nullptr, nullptr, nullptr, fn);
    return launch_score(h, xs, zs, m, acq, out, nullptr, nullptr, nullptr, fn);
  };
  if (!h->fitted) { set_error("vzgp_eagle_run before vzgp_fit"); return VZGP_ERR_STATE; }
  VZ_ARG(best_x != nullptr || h->dc == 0, "best_x");
  VZ_ARG(best_z != nullptr || h->dk == 0, "best_z");
  VZ_TRY(eagle_check_config(h, cfg, count));
  VZ_ARG(cfg->n_parallel <= 1, "n_parallel > 1 runs through the host-stepped loop (vzgp_eagle_begin ...)");
  VZ_ARG(n_prior >= 0, "n_prior");
  VZ_ARG(n_prior == 0 || prior != nullptr || h->dc == 0, "prior");
  VZ_ARG(n_prior == 0 || prior_z != nullptr || h->dk == 0, "prior_z");
  Guard g(h->device);
  const int B = cfg->batch_size, D = h->dc, Dk = h->dk;
  EagleDev e;
  EagleScratch es;
  VZ_TRY(eagle_setup(h, cfg, cat_sizes, count, seed, n_prior, &e, &es));
  double* prior_r = es.prior_r;
  double* chosen_r = es.chosen_r;
  int* ord = es.ord;
  if (scal) VZ_TRY(prepare_scalarization(h, scal));
  if (pem) VZ_TRY(prepare_score_pe_multi(h, pem));
  VZ_TRY(launch_eagle_init(h, e));
  if (n_prior > 0) {
    VZ_TRY(score_batch(prior, Dk > 0 ? prior_z : nullptr, n_prior, prior_r));
    VZ_TRY(launch_eagle_seed_priors(h, e, prior, prior_z, prior_r, n_prior, ord, chosen_r));
  }
  const int steps = (cfg->max_evaluations - 1) / B + 1;
  auto one_step = [&]() -> int {
    VZ_TRY(launch_eagle_suggest(h, e));
    VZ_TRY(score_batch(e.batch, Dk > 0 ? e.batch_z : nullptr, B, e.batch_r));
    VZ_TRY(launch_eagle_update(h, e));
    return 0;
  };
  // Step 0 runs eagerly (it sizes every workspace); the remaining steps replay one captured
  // CUDA graph of the suggest -> score -> update sequence: the iteration counter and all state
  // live in device memory, so the launches are identical and the host only enqueues graphs.
  bool done = false;
  // the persistent and cooperative forms evaluate single-metric acquisitions only
  const bool fused_ok = n_ens <= 1 && !scal && !stack_alphas && !pem;
  if (fused_ok && eagle_persistent_eligible(h, pe ? hB : nullptr, e)) {
    // small study: the whole loop is one persistent single-CTA kernel
    VZ_TRY(launch_eagle_persistent64(h, pe ? hB : nullptr, e, acq, pe, steps, fn));
    done = true;
  } else if (fused_ok && eagle_grid_eligible(h, pe ? hB : nullptr, e)) {
    // mid-size study: one cooperative launch, phases separated by grid barriers.  If the cooperative
    // launch is refused (nothing has run then) the launch-per-phase loop below takes over.
    done = launch_eagle_grid(h, pe ? hB : nullptr, e, acq, pe, steps, fn) == 0;
    if (!done) cudaGetLastError();
  }
  if (!done) {
  VZ_TRY(one_step());
  if (steps > 1) {
    const int64_t l0 = h->launches;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    VZ_CUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeRelaxed));
    int st = one_step();
    cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
    if (st < 0 || ce != cudaSuccess || graph == nullptr) {
      if (graph) cudaGraphDestroy(graph);
      if (st >= 0) set_error("eagle: stream capture failed: %s", cudaGetErrorString(ce));
      return st < 0 ? st : VZGP_ERR_CUDA;
    }
    const int64_t per_step = h->launches - l0;
    ce = cudaGraphInstantiate(&exec, graph, 0);
    if (ce != cudaSuccess) {
      cudaGraphDestroy(graph);
      set_error("eagle: cudaGraphInstantiate: %s", cudaGetErrorString(ce));
      return VZGP_ERR_CUDA;
    }
    h->launches = l0;  // the capture itself executed nothing
    for (int t = 1; t < steps; ++t) {
      ce = cudaGraphLaunch(exec, h->stream);
      if (ce != cudaSuccess) break;
      h->launches += per_step;
    }
    cudaGraphExecDestroy(exec);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
      set_error("eagle: cudaGraphLaunch: %s", cudaGetErrorString(ce));
      return VZGP_ERR_CUDA;
    }
  }
  }
  if (D > 0) VZ_CUDA(cudaMemcpyAsync(best_x, e.best_x, sizeof(double) * (size_t)count * D, cudaMemcpyDeviceToHost, h->stream));
  if (Dk > 0) VZ_CUDA(cudaMemcpyAsync(best_z, e.best_z, sizeof(int32_t) * (size_t)count * Dk, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(best_score, e.best_r, sizeof(double) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

// ---- host-stepped Eagle loop: same state and kernels, the caller scores every batch -----------------
struct EagleStepState {
  EagleDev e;
  EagleScratch es;
  int n_prior = 0;
  bool seeded = false, asked = false;
};
static EagleStepState* step_state(vzgp_handle* h) { return static_cast<EagleStepState*>(h->eagle_step); }
static void eagle_step_free(vzgp_handle* h) {
  if (h->eagle_step) { delete step_state(h); h->eagle_step = nullptr; }
}

int vzgp_eagle_begin(vzgp_handle* h, const vzgp_eagle_config* cfg, const int32_t* cat_sizes, int count, uint64_t seed,
                     int n_prior, double** prior_rewards_dev) {
  VZ_ARG(h && cfg, "handle / cfg");
  VZ_ARG(h->dc + h->dk > 0, "the handle needs its feature dimensions (fit a model first)");
  VZ_TRY(eagle_check_config(h, cfg, count));
  VZ_ARG(n_prior >= 0, "n_prior");
  Guard g(h->device);
  if (h->eagle_step) { delete step_state(h); h->eagle_step = nullptr; }
  EagleStepState* st = new EagleStepState();
  int rc = eagle_setup(h, cfg, cat_sizes, count, seed, n_prior, &st->e, &st->es);
  if (rc == 0) rc = launch_eagle_init(h, st->e);
  if (rc < 0) { delete st; return rc; }
  st->n_prior = n_prior;
  h->eagle_step = st;
  if (prior_rewards_dev) *prior_rewards_dev = st->es.prior_r;
  return 0;
}

int vzgp_eagle_seed(vzgp_handle* h, const double* prior, const int32_t* prior_z) {
  VZ_ARG(h && h->eagle_step, "vzgp_eagle_begin first");
  EagleStepState* st = step_state(h);
  VZ_ARG(st->n_prior > 0 && !st->seeded && !st->asked, "seeding happens once, before the first ask, with n_prior > 0");
  VZ_ARG(prior != nullptr || h->dc == 0, "prior");
  VZ_ARG(prior_z != nullptr || h->dk == 0, "prior_z");
  Guard g(h->device);
  VZ_TRY(launch_eagle_seed_priors(h, st->e, prior, prior_z, st->es.prior_r, st->n_prior, st->es.ord, st->es.chosen_r));
  st->seeded = true;
  return 0;
}

int vzgp_eagle_ask(vzgp_handle* h, const double** batch_x_dev, const int32_t** batch_z_dev, double** batch_rewards_dev) {
  VZ_ARG(h && h->eagle_step, "vzgp_eagle_begin first");
  EagleStepState* st = step_state(h);
  VZ_ARG(!st->asked, "vzgp_eagle_tell the previous batch first");
  Guard g(h->device);
  VZ_TRY(launch_eagle_suggest(h, st->e));
  st->asked = true;
  if (batch_x_dev) *batch_x_dev = st->e.batch;
  if (batch_z_dev) *batch_z_dev = st->e.batch_z;
  if (batch_rewards_dev) *batch_rewards_dev = st->e.batch_r;
  return 0;
}

int vzgp_eagle_tell(vzgp_handle* h) {
  VZ_ARG(h && h->eagle_step, "vzgp_eagle_begin first");
  EagleStepState* st = step_state(h);
  VZ_ARG(st->asked, "vzgp_eagle_ask first");
  Guard g(h->device);
  VZ_TRY(launch_eagle_update(h, st->e));
  st->asked = false;
  return 0;
}

int vzgp_eagle_end(vzgp_handle* h, double* best_x, int32_t* best_z, double* best_score) {
  VZ_ARG(h && h->eagle_step && best_score, "vzgp_eagle_begin first / best_score");
  EagleStepState* st = step_state(h);
  VZ_ARG(best_x != nullptr || h->dc == 0, "best_x");
  VZ_ARG(best_z != nullptr || h->dk == 0, "best_z");
  Guard g(h->device);
  const EagleDev& e = st->e;
  const int count = e.count, D = e.D, Dk = e.Dk;
  if (D > 0) VZ_CUDA(cudaMemcpyAsync(best_x, e.best_x, sizeof(double) * (size_t)count * D, cudaMemcpyDeviceToHost, h->stream));
  if (Dk > 0) VZ_CUDA(cudaMemcpyAsync(best_z, e.best_z, sizeof(int32_t) * (size_t)count * Dk, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(best_score, e.best_r, sizeof(double) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  delete st;
  h->eagle_step = nullptr;
  return 0;
}

int vzgp_eagle_run(vzgp_handle* h, const vzgp_eagle_config* cfg, const vzgp_acq* acq, const double* prior,
                   const int32_t* prior_z, int n_prior, const int32_t* cat_sizes, int count, uint64_t seed,
                   double* best_x, int32_t* best_z, double* best_score) {
  VZ_ARG(acq != nullptr, "acq");
  return eagle_run_impl(h, nullptr, cfg, acq, nullptr, prior, prior_z, n_prior, cat_sizes, count, seed, best_x,
                        best_z, best_score);
}

int vzgp_eagle_run_multi(vzgp_handle* h, const vzgp_eagle_config* cfg, const vzgp_scalarization* sc,
                         const double* prior, const int32_t* prior_z, int n_prior, const int32_t* cat_sizes,
                         int count, uint64_t seed, double* best_x, int32_t* best_z, double* best_score) {
  VZ_ARG(sc != nullptr, "scalarization");
  return eagle_run_impl(h, nullptr, cfg, nullptr, nullptr, prior, prior_z, n_prior, cat_sizes, count, seed, best_x,
                        best_z, best_score, nullptr, 0, sc);
}

int vzgp_score_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_scalarization* sc,
                     double* score, double* mu, double* sigma) {
  VZ_ARG(h != nullptr && sc != nullptr, "handle / scalarization");
  if (!h->fitted) { set_error("vzgp_score_multi before vzgp_fit_multi"); return VZGP_ERR_STATE; }
  VZ_ARG(M >= 0 && (M == 0 || score != nullptr), "M / score");
  VZ_ARG(M == 0 || Xs != nullptr || h->dc == 0, "Xs");
  VZ_ARG(M == 0 || Zs != nullptr || h->dk == 0, "Zs");
  Guard g(h->device);
  VZ_TRY(prepare_scalarization(h, sc));
  return launch_score_multi(h, Xs, Zs, M, score, mu, sigma);
}

static int check_pe(vzgp_handle* hA, vzgp_handle* hB, const vzgp_pe_params* pe) {
  VZ_ARG(hA && hB && pe, "handles / pe");
  if (!hA->fitted || !hB->fitted) { set_error("GP-UCB-PE scoring needs both models fitted"); return VZGP_ERR_STATE; }
  VZ_ARG(hA->device == hB->device && hA->stream == hB->stream, "both models must share device and stream");
  VZ_ARG(hA->dc == hB->dc && hA->dk == hB->dk, "both models must have the same feature dimensions");
  VZ_ARG(pe->mode == 0 || pe->mode == 1, "mode");
  return 0;
}

int vzgp_score_pe(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                  const vzgp_pe_params* pe, double* score, double* mu, double* sigma, double* sigma_all) {
  VZ_TRY(check_pe(hA, hB, pe));
  VZ_ARG(M >= 0 && (M == 0 || score != nullptr), "M / score");
  Guard g(hA->device);
  return launch_score_pe(hA, hB, Xs, Zs, M, pe, score, mu, sigma, sigma_all);
}

int vzgp_score_set_pe(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, int n_sets, int q, const vzgp_pe_params* pe,
                      double* score, double* mu, double* sigma, double* sigma_all) {
  VZ_TRY(check_pe(hA, hB, pe));
  VZ_ARG(hA->dk == 0, "set acquisitions: continuous features only");
  VZ_ARG(n_sets >= 0 && q >= 1 && q <= 16, "n_sets >= 0, 1 <= q <= 16");
  VZ_ARG(n_sets == 0 || (Xs != nullptr && score != nullptr), "Xs / score");
  if (n_sets == 0) return 0;
  Guard g(hA->device);
  const int M = n_sets * q;
  // pe_tmp of A: mu_a | sd_a | linf_b | dummy_a | dummy_b | sd_b [6 M]  then  cov [M x M]  then  mean_b [M]
  VZ_TRY(hA->pe_tmp.reserve(sizeof(double) * (7 * (size_t)M + (size_t)M * M)));
  double* t = hA->pe_tmp.as<double>();
  double* mu_a = mu ? mu : t;
  double* sd_a = sigma ? sigma : t + M;
  double* linf_b = t + 2 * (size_t)M;
  double* dummy_a = t + 3 * (size_t)M;
  double* dummy_b = t + 4 * (size_t)M;
  double* sd_b = t + 5 * (size_t)M;
  double* mean_b = t + 6 * (size_t)M;
  double* cov = t + 7 * (size_t)M;
  const vzgp_acq none = posterior_request(), accb = posterior_request(pe->tr_dim_mask, pe->tr_rows);
  VZ_TRY(launch_score(hA, Xs, nullptr, M, &none, dummy_a, mu_a, sd_a, nullptr));
  const bool want_tr = tr_needs_distance(trust_region_of(hB, *pe, true));
  if (want_tr) VZ_TRY(launch_score(hB, Xs, nullptr, M, &accb, dummy_b, nullptr, sd_b, linf_b));
  VZ_TRY(vzgp_posterior_multi(hB, Xs, nullptr, M, 1, mean_b, cov, M));
  return launch_set_pe_combine(hA, n_sets, q, pe, cov, M, mu_a, sd_a, want_tr ? linf_b : nullptr, score, sigma_all);
}

int vzgp_eagle_run_pe(vzgp_handle* hA, vzgp_handle* hB, const vzgp_eagle_config* cfg,
                      const vzgp_pe_params* pe, const double* prior, const int32_t* prior_z, int n_prior,
                      const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                      double* best_score) {
  VZ_TRY(check_pe(hA, hB, pe));
  return eagle_run_impl(hA, hB, cfg, nullptr, pe, prior, prior_z, n_prior, cat_sizes, count, seed, best_x, best_z,
                        best_score);
}

static int check_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const vzgp_pe_multi_params* pe) {
  VZ_ARG(hA && hB && pe, "handles / pe");
  if (!hA->fitted || !hB->fitted) { set_error("GP-UCB-PE scoring needs both models fitted"); return VZGP_ERR_STATE; }
  VZ_ARG(hA->device == hB->device && hA->stream == hB->stream, "both models must share device and stream");
  VZ_ARG(hA->dc == hB->dc && hA->dk == hB->dk, "both models must have the same feature dimensions");
  VZ_ARG(pe->mode == 0 || pe->mode == 1, "mode");
  VZ_ARG(pe->n_metrics >= 1 && pe->n_metrics <= kMaxMetrics, "1 <= n_metrics <= 8");
  VZ_ARG(pe->n_metrics == hA->n_metrics, "n_metrics must equal the metrics model A was fitted with (vzgp_fit_multi)");
  VZ_ARG(pe->mode != 1 || pe->thresholds != nullptr, "thresholds (mode 1)");
  VZ_ARG(pe->mode != 1 || (pe->region_penalty >= VZGP_REGION_AVERAGE && pe->region_penalty <= VZGP_REGION_INTERSECTION),
         "region_penalty");
  VZ_ARG(pe->mode != 0 || pe->scalarization != nullptr, "scalarization (mode 0)");
  return 0;
}

int vzgp_score_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const double* Xs, const int32_t* Zs, int M,
                        const vzgp_pe_multi_params* pe, double* score, double* mu, double* sigma, double* sigma_all) {
  VZ_TRY(check_pe_multi(hA, hB, pe));
  VZ_ARG(M >= 0 && (M == 0 || score != nullptr), "M / score");
  VZ_ARG(M == 0 || Xs != nullptr || hA->dc == 0, "Xs");
  VZ_ARG(M == 0 || Zs != nullptr || hA->dk == 0, "Zs");
  Guard g(hA->device);
  VZ_TRY(prepare_score_pe_multi(hA, pe));
  return launch_score_pe_multi(hA, hB, Xs, Zs, M, pe, score, mu, sigma, sigma_all);
}

int vzgp_eagle_run_pe_multi(vzgp_handle* hA, vzgp_handle* hB, const vzgp_eagle_config* cfg,
                            const vzgp_pe_multi_params* pe, const double* prior, const int32_t* prior_z, int n_prior,
                            const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                            double* best_score) {
  VZ_TRY(check_pe_multi(hA, hB, pe));
  return eagle_run_impl(hA, hB, cfg, nullptr, nullptr, prior, prior_z, n_prior, cat_sizes, count, seed, best_x, best_z,
                        best_score, nullptr, 0, nullptr, nullptr, pe);
}

static int check_ensemble(vzgp_handle* const* hs, int E) {
  VZ_ARG(hs != nullptr && E >= 1 && E <= 16, "1 <= E <= 16 handles");
  for (int e = 0; e < E; ++e) {
    VZ_ARG(hs[e] != nullptr, "handle");
    if (!hs[e]->fitted) { set_error("ensemble scoring needs every member fitted"); return VZGP_ERR_STATE; }
    VZ_ARG(hs[e]->device == hs[0]->device && hs[e]->stream == hs[0]->stream, "members must share device and stream");
    VZ_ARG(hs[e]->dc == hs[0]->dc && hs[e]->dk == hs[0]->dk && hs[e]->n_valid == hs[0]->n_valid,
           "members must be fitted on the same trials");
  }
  return 0;
}

int vzgp_score_ensemble(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int M,
                        const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf) {
  VZ_TRY(check_ensemble(hs, E));
  VZ_ARG(acq != nullptr, "acq");
  VZ_ARG(M >= 0 && (M == 0 || score != nullptr), "M / score");
  VZ_ARG(M == 0 || Xs != nullptr || hs[0]->dc == 0, "Xs");
  VZ_ARG(M == 0 || Zs != nullptr || hs[0]->dk == 0, "Zs");
  Guard g(hs[0]->device);
  return launch_score_ensemble(hs, E, Xs, Zs, M, acq, score, mu, sigma, linf, handle_acq(hs[0]));
}

int vzgp_eagle_run_ensemble(vzgp_handle* const* hs, int E, const vzgp_eagle_config* cfg, const vzgp_acq* acq,
                            const double* prior, const int32_t* prior_z, int n_prior, const int32_t* cat_sizes,
                            int count, uint64_t seed, double* best_x, int32_t* best_z, double* best_score) {
  VZ_TRY(check_ensemble(hs, E));
  VZ_ARG(acq != nullptr, "acq");
  return eagle_run_impl(hs[0], nullptr, cfg, acq, nullptr, prior, prior_z, n_prior, cat_sizes, count, seed, best_x,
                        best_z, best_score, hs, E);
}

static int check_qacq(const vzgp_qacq* qa, int n_sets, int q) {
  VZ_ARG(qa != nullptr, "qacq");
  VZ_ARG(qa->kind == VZGP_QACQ_QEI || qa->kind == VZGP_QACQ_QPI || qa->kind == VZGP_QACQ_QUCB, "kind");
  VZ_ARG(q >= 1 && q <= 16, "1 <= q <= 16");
  VZ_ARG(qa->num_samples >= 1 && qa->num_samples <= 8192, "1 <= num_samples <= 8192");
  VZ_ARG(n_sets >= 0 && (int64_t)n_sets * q <= INT_MAX / 16, "n_sets");
  return 0;
}

int vzgp_score_qsets(vzgp_handle* const* hs, int E, const double* Xs, const int32_t* Zs, int n_sets, int q,
                     const vzgp_qacq* qa, uint64_t seed, double* score, double* mu, double* sigma, double* linf) {
  VZ_TRY(check_ensemble(hs, E));
  VZ_TRY(check_qacq(qa, n_sets, q));
  for (int e = 0; e < E; ++e) VZ_ARG(hs[e]->n_metrics == 1, "q-acquisitions: single-metric models");
  VZ_ARG(hs[0]->dc <= kMaxDc && hs[0]->dk <= kMaxDk, "Dc <= 64, Dk <= 32");
  VZ_ARG(n_sets == 0 || score != nullptr, "score");
  VZ_ARG(n_sets == 0 || Xs != nullptr || hs[0]->dc == 0, "Xs");
  VZ_ARG(n_sets == 0 || Zs != nullptr || hs[0]->dk == 0, "Zs");
  if (n_sets == 0) return 0;
  Guard g(hs[0]->device);
  return launch_score_qsets(hs, E, Xs, Zs, n_sets, q, qa, seed, score, mu, sigma, linf);
}

int vzgp_qacq_from_moments(vzgp_handle* h, int n_sets, int q, int E, const double* mean, const double* cov,
                           const vzgp_qacq* qa, uint64_t seed, double* score) {
  VZ_ARG(h != nullptr, "handle");
  VZ_ARG(E >= 1 && E <= 16, "1 <= E <= 16");
  VZ_TRY(check_qacq(qa, n_sets, q));
  VZ_ARG(n_sets == 0 || (mean != nullptr && cov != nullptr && score != nullptr), "mean / cov / score");
  if (n_sets == 0) return 0;
  Guard g(h->device);
  return launch_qacq_mc(h, n_sets, q, E, mean, cov, nullptr, qa, seed, score, nullptr, nullptr);
}

static int check_stack(vzgp_handle* const* hs, int E, const double* alphas) {
  VZ_ARG(hs != nullptr && alphas != nullptr && E >= 1 && E <= 16, "1 <= E <= 16 handles, alphas");
  for (int e = 0; e < E; ++e) {
    VZ_ARG(hs[e] != nullptr, "handle");
    if (!hs[e]->fitted) { set_error("stacked scoring needs every level fitted"); return VZGP_ERR_STATE; }
    VZ_ARG(hs[e]->device == hs[0]->device && hs[e]->stream == hs[0]->stream, "levels must share device and stream");
    VZ_ARG(hs[e]->dc == hs[0]->dc && hs[e]->dk == hs[0]->dk, "levels must have the same feature dimensions");
    VZ_ARG(e == 0 || (alphas[e] >= 0.0 && alphas[e] <= 1.0), "0 <= alpha <= 1");
  }
  return 0;
}

int vzgp_score_stack(vzgp_handle* const* hs, int E, const double* alphas, const double* Xs, const int32_t* Zs, int M,
                     const vzgp_acq* acq, double* score, double* mu, double* sigma, double* linf) {
  VZ_TRY(check_stack(hs, E, alphas));
  VZ_ARG(acq != nullptr, "acq");
  VZ_ARG(M >= 0 && (M == 0 || score != nullptr), "M / score");
  VZ_ARG(M == 0 || Xs != nullptr || hs[0]->dc == 0, "Xs");
  VZ_ARG(M == 0 || Zs != nullptr || hs[0]->dk == 0, "Zs");
  Guard g(hs[0]->device);
  return launch_score_stack(hs, E, alphas, Xs, Zs, M, acq, score, mu, sigma, linf, handle_acq(hs[0]));
}

int vzgp_eagle_run_stack(vzgp_handle* const* hs, int E, const double* alphas, const vzgp_eagle_config* cfg,
                         const vzgp_acq* acq, const double* prior, const int32_t* prior_z, int n_prior,
                         const int32_t* cat_sizes, int count, uint64_t seed, double* best_x, int32_t* best_z,
                         double* best_score) {
  VZ_TRY(check_stack(hs, E, alphas));
  VZ_ARG(acq != nullptr, "acq");
  return eagle_run_impl(hs[E - 1], nullptr, cfg, acq, nullptr, prior, prior_z, n_prior, cat_sizes, count, seed, best_x,
                        best_z, best_score, hs, E, nullptr, alphas);
}

int vzgp_nll_grad_batch(vzgp_handle* const* hs, int R, const double* X, const int32_t* Z, const double* Y, int N,
                        int Dc, int Dk, int n_valid, int n_metrics, const vzgp_params* ps, const uint8_t* active,
                        double* loss_out, double* grad_out, int* status_out) {
  VZ_ARG(hs && ps && loss_out && grad_out && status_out, "pointers");
  VZ_ARG(R >= 1 && R <= kMaxBatch, "1 <= R <= 16");
  VZ_ARG(N > kBlk, "the batched evaluation is for N > 64 (smaller studies: vzgp_nll_grad per restart)");
  for (int r = 0; r < R; ++r) VZ_ARG(ps[r].linear_coef == 0.0, "linear_coef models take vzgp_nll_grad per restart");
  VZ_ARG(n_valid >= 1 && n_valid <= N, "1 <= n_valid <= N");
  VZ_ARG(n_metrics >= 1 && n_metrics <= kMaxMetrics, "1 <= n_metrics <= 8");
  VZ_ARG(X != nullptr || Dc == 0, "X");
  VZ_ARG(Z != nullptr || Dk == 0, "Z");
  VZ_ARG(Y != nullptr, "Y");
  for (int r = 0; r < R; ++r) {
    VZ_ARG(hs[r] != nullptr && hs[r]->device == hs[0]->device, "handles must live on one device");
    for (int q = 0; q < r; ++q) VZ_ARG(hs[q] != hs[r] && hs[q]->stream != hs[r]->stream, "handles need distinct streams");
  }
  vzgp_handle* lead = hs[0];
  Guard g(lead->device);
  const int np = round_up(N, kBlk), nq = Dc + Dk + 2;
  const size_t res_bytes = sizeof(double) * (2 + nq) + sizeof(int) * 2;
  if (!lead->batch) lead->batch = new BatchGraph();
  BatchGraph* b = static_cast<BatchGraph*>(lead->batch);
  KernelParams kps[kMaxBatch];
  for (int r = 0; r < R; ++r) VZ_TRY(fill_kernel_params(&ps[r], Dc, Dk, &kps[r]));
  // ---- is the captured graph still valid? ----
  bool hit = b->exec && b->key_ptr[0] == X && b->key_ptr[1] == Z && b->key_ptr[2] == Y && b->key_dims[0] == N &&
             b->key_dims[1] == Dc && b->key_dims[2] == Dk && b->key_dims[3] == n_valid && b->key_dims[4] == n_metrics &&
             b->key_dims[5] == R;
  for (int r = 0; hit && r < R; ++r) {
    const void* cur[kNllBufs];
    handle_bufs(hs[r], cur);
    hit = b->hs[r] == hs[r] && hs[r]->df_nb[1] == np / 64;
    for (int q = 0; hit && q < kNllBufs; ++q) hit = cur[q] == b->bufs[r][q];
  }
  if (!hit) {
    batch_drop(b);
    if (!b->fork) {
      VZ_CUDA(cudaEventCreateWithFlags(&b->fork, cudaEventDisableTiming));
      for (int r = 0; r < kMaxBatch; ++r) VZ_CUDA(cudaEventCreateWithFlags(&b->join[r], cudaEventDisableTiming));
    }
    for (int r = 0; r < R; ++r) {
      vzgp_handle* h = hs[r];
      VZ_TRY(ensure_model_buffers(h, np, Dc, Dk, n_metrics));
      VZ_TRY(h->Kinv.reserve(sizeof(double) * (size_t)np * np * kLauumSplit));
      VZ_TRY(h->Tws.reserve(sizeof(double) * (size_t)np * np));
      VZ_TRY(chol_dataflow_prepare(h, np, true));
      VZ_TRY(ensure_pinned(h, res_bytes));
      h->fitted = false; h->i8_ready = false;
      h->n = N; h->np = np; h->dc = Dc; h->dk = Dk; h->n_valid = n_valid; h->n_metrics = n_metrics;
      h->mean_const = 0.0;   // captured by the label-padding node (see nll_graph_eval)
      VZ_CUDA(cudaStreamSynchronize(h->stream));
    }
    const int64_t l0[kMaxBatch] = {};
    int64_t before[kMaxBatch];
    for (int r = 0; r < R; ++r) before[r] = hs[r]->launches;
    (void)l0;
    if (cudaStreamBeginCapture(lead->stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) { cudaGetLastError(); set_error("batch capture refused"); return VZGP_ERR_CUDA; }
    int st = 0;
    cudaEventRecord(b->fork, lead->stream);
    for (int r = 1; r < R; ++r) cudaStreamWaitEvent(hs[r]->stream, b->fork, 0);
    for (int r = 0; r < R && st >= 0; ++r) {
      vzgp_handle* h = hs[r];
      st = nll_sequence(h, X, Z, Y, N, Dc, Dk, n_valid, kps[r], ps[r].observation_noise_variance, n_metrics);
      if (st < 0) break;
      char* pin = static_cast<char*>(h->pinned);
      cudaMemcpyAsync(pin, h->small.as<char>() + kOffLogdet, sizeof(double) * 2, cudaMemcpyDeviceToHost, h->stream);
      cudaMemcpyAsync(pin + 16, h->small.as<char>() + kOffGrad, sizeof(double) * nq, cudaMemcpyDeviceToHost, h->stream);
      cudaMemcpyAsync(pin + 16 + sizeof(double) * nq, h->small.as<char>() + kOffFlag, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
      if (r > 0) { cudaEventRecord(b->join[r], h->stream); cudaStreamWaitEvent(lead->stream, b->join[r], 0); }
    }
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(lead->stream, &graph);
    b->launches = 0;
    for (int r = 0; r < R; ++r) { b->launches += (int)(hs[r]->launches - before[r]); hs[r]->launches = before[r]; }
    if (st < 0 || ce != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      if (st >= 0) set_error("batch capture failed: %s", cudaGetErrorString(ce));
      cudaGetLastError();
      return st < 0 ? st : VZGP_ERR_CUDA;
    }
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) { cudaGraphDestroy(graph); cudaGetLastError(); set_error("cudaGraphInstantiate (batch)"); return VZGP_ERR_CUDA; }
    size_t nn = 0;
    cudaGraphGetNodes(graph, nullptr, &nn);
    std::vector<cudaGraphNode_t> nodes(nn);
    cudaGraphGetNodes(graph, nodes.data(), &nn);
    const void* want[3] = {kernel_matrix_func(), transpose_scale_func(), nll_grad_tiles_func()};
    const int id_arg[3] = {6, 4, 5};       // output / workspace pointer that tells the R branches apart
    for (int r = 0; r < R; ++r) for (int q = 0; q < 3; ++q) b->nodes[r][q] = nullptr;
    for (size_t i = 0; i < nn; ++i) {
      cudaGraphNodeType ty;
      if (cudaGraphNodeGetType(nodes[i], &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
      cudaKernelNodeParams kpar;
      if (cudaGraphKernelNodeGetParams(nodes[i], &kpar) != cudaSuccess) continue;
      for (int q = 0; q < 3; ++q) {
        if (kpar.func != want[q]) continue;
        const void* idp = *static_cast<const void* const*>(kpar.kernelParams[id_arg[q]]);
        for (int r = 0; r < R; ++r) {
          const void* mine = q == 0 ? hs[r]->Kws.ptr : (q == 1 ? hs[r]->XT.ptr : hs[r]->Kinv.ptr);
          if (idp == mine) b->nodes[r][q] = nodes[i];
        }
      }
    }
    cudaGetLastError();
    for (int r = 0; r < R; ++r)
      if (!b->nodes[r][0] || (Dc > 0 && !b->nodes[r][1]) || !b->nodes[r][2]) {
        cudaGraphExecDestroy(exec); cudaGraphDestroy(graph);
        set_error("batch graph: kernel nodes of restart %d not found", r);
        return VZGP_ERR_CUDA;
      }
    b->graph = graph; b->exec = exec;
    b->key_ptr[0] = X; b->key_ptr[1] = Z; b->key_ptr[2] = Y;
    b->key_dims[0] = N; b->key_dims[1] = Dc; b->key_dims[2] = Dk; b->key_dims[3] = n_valid; b->key_dims[4] = n_metrics; b->key_dims[5] = R;
    for (int r = 0; r < R; ++r) { b->hs[r] = hs[r]; handle_bufs(hs[r], b->bufs[r]); }
  }
  // ---- this round's hyper-parameters, launch, wait ----
  const int arg_idx[3] = {kKernelMatrixKpArg, kTransposeScaleKpArg, kNllGradTilesKpArg};
  const int arg_cnt[3] = {kKernelMatrixArgs, kTransposeScaleArgs, kNllGradTilesArgs};
  double sn2s[kMaxBatch];
  for (int r = 0; r < R; ++r) {
    if (active && !active[r]) continue;
    sn2s[r] = ps[r].observation_noise_variance;
    hs[r]->kp = kps[r]; hs[r]->sn2 = sn2s[r]; hs[r]->mean_const = 0.0; hs[r]->fitted = false; hs[r]->i8_ready = false;
    for (int q = 0; q < 3; ++q) {
      if (!b->nodes[r][q]) continue;
      cudaKernelNodeParams kpar;
      VZ_CUDA(cudaGraphKernelNodeGetParams(b->nodes[r][q], &kpar));
      void* args[16];
      for (int a2 = 0; a2 < arg_cnt[q]; ++a2) args[a2] = kpar.kernelParams[a2];
      args[arg_idx[q]] = &kps[r];
      if (q == 0) args[kKernelMatrixDiagArg] = &sn2s[r];
      kpar.kernelParams = args;
      VZ_CUDA(cudaGraphExecKernelNodeSetParams(b->exec, b->nodes[r][q], &kpar));
    }
  }
  VZ_CUDA(cudaGraphLaunch(b->exec, lead->stream));
  lead->launches += b->launches;
  VZ_CUDA(cudaStreamSynchronize(lead->stream));
  for (int r = 0; r < R; ++r) {
    status_out[r] = 0;
    if (active && !active[r]) continue;
    const char* pin = static_cast<const char*>(hs[r]->pinned);
    const double* h2 = reinterpret_cast<const double*>(pin);
    const double* hg = reinterpret_cast<const double*>(pin + 16);
    const int bad = *reinterpret_cast<const int*>(pin + 16 + sizeof(double) * nq);
    if (!bad) {
      hs[r]->nll_route = VZGP_NLL_BATCH; hs[r]->factor_route = hs[r]->nll_factor_route;
      finish_loss(&ps[r], Dc, Dk, n_valid, n_metrics, h2[1] + h2[0], hg, loss_out + r, grad_out + (size_t)r * nq);
    } else {
      // a pivot failed without jitter: this restart alone takes the path with the retry loop
      status_out[r] = vzgp_nll_grad_multi(hs[r], X, Z, Y, N, Dc, Dk, n_valid, n_metrics, &ps[r], loss_out + r, grad_out + (size_t)r * nq);
      if (status_out[r] < 0) return status_out[r];
    }
  }
  return 0;
}

int vzgp_posterior(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, int add_noise,
                   double* mean, double* cov, int ldc) {
  return vzgp_posterior_multi(h, Xs, Zs, M, add_noise, mean, cov, ldc);
}

int vzgp_posterior_multi(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, int add_noise,
                         double* mean, double* cov, int ldc) {
  VZ_ARG(h && mean && cov, "handle / outputs");
  if (!h->fitted) { set_error("vzgp_posterior before vzgp_fit"); return VZGP_ERR_STATE; }
  VZ_ARG(M >= 1 && ldc >= M, "M, ldc");
  VZ_ARG(Xs != nullptr || h->dc == 0, "Xs");
  Guard g(h->device);
  const int np = h->np, mp = round_up(M, kBlk);
  // layout in Kinv buffer: Ks [mp x np] | W [mp x np] | C [mp x mp] | Xs padded [mp x dc] | mean [mp]
  const size_t nks = (size_t)mp * np, nc = (size_t)mp * mp, nx = (size_t)mp * (h->dc > 0 ? h->dc : 1);
  const int nm = h->n_metrics;
  VZ_TRY(h->Kinv.reserve(sizeof(double) * (2 * nks + nc + nx + (size_t)mp * nm) + sizeof(int32_t) * (size_t)mp * (h->dk > 0 ? h->dk : 1)));
  double* Ks = h->Kinv.as<double>();
  double* W = Ks + nks;
  double* C = W + nks;
  double* Xp = C + nc;
  double* mu = Xp + nx;
  int32_t* Zp = reinterpret_cast<int32_t*>(mu + (size_t)mp * nm);
  VZ_CUDA(cudaMemsetAsync(Ks, 0, sizeof(double) * nks, h->stream));
  if (h->dc > 0) VZ_TRY(launch_pad_rows(h, Xs, M, h->dc, mp, Xp));
  if (h->dk > 0) VZ_TRY(launch_pad_rows_i32(h, Zs, M, h->dk, mp, Zp));
  VZ_TRY(launch_cross_kernel(h, Xp, Zp, M, h->X.as<double>(), h->Z.as<int32_t>(), np, h->n_valid, h->kp, Ks, np));
  VZ_TRY(launch_cross_kernel(h, Xp, Zp, mp, Xp, Zp, mp, mp, h->kp, C, mp));
  VZ_TRY(launch_gemm_nt_tri(h, Ks, np, mp, h->Linv.as<double>(), np, np, W, np));
  VZ_TRY(launch_cov_update(h, W, np, np, mp, C, mp, add_noise ? h->sn2 : 0.0));
  for (int m = 0; m < nm; ++m)
    VZ_TRY(launch_gemv_rows(h, Ks, np, mp, h->alpha.as<double>() + (size_t)m * np, mu + (size_t)m * mp, 0, np));
  if (h->mean_const != 0.0) VZ_TRY(launch_add_scalar(h, (int)((size_t)mp * nm), h->mean_const, mu));
  VZ_CUDA(cudaMemcpy2DAsync(cov, sizeof(double) * ldc, C, sizeof(double) * mp, sizeof(double) * M, M,
                            cudaMemcpyDeviceToDevice, h->stream));
  VZ_CUDA(cudaMemcpy2DAsync(mean, sizeof(double) * M, mu, sizeof(double) * mp, sizeof(double) * M, nm,
                            cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

int vzgp_score_topk(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                    int count, double* score_dev, double* best_x, double* best_score, int64_t* best_index) {
  VZ_ARG(best_x && best_score, "outputs");
  VZ_ARG(M >= 1, "M >= 1");
  Guard g(h ? h->device : 0);
  const int dc = h ? h->dc : 0;
  double* dS = score_dev;
  if (!dS) {
    VZ_ARG(h != nullptr, "handle");
    VZ_TRY(h->out_dev.reserve(sizeof(double) * ((size_t)M + (size_t)kMaxTopk * (dc > 0 ? dc : 1))));
    dS = h->out_dev.as<double>();
  }
  VZ_TRY(check_scoring(h, Xs, Zs, M, acq, dS));
  VZ_ARG(h->dk == 0, "continuous features only");
  VZ_TRY(h->xs_dev.reserve(0));
  VZ_TRY(launch_score(h, Xs, Zs, M, acq, dS, nullptr, nullptr, nullptr, handle_acq(h)));
  long long* d_idx; double* d_val;
  VZ_TRY(topk_to_device(h, dS, M, count, &d_idx, &d_val));
  double* dBest = reinterpret_cast<double*>(h->small.as<char>() + kOffRows);
  VZ_ARG((size_t)count * dc * sizeof(double) <= kRowsBytes, "count * Dc too large");
  VZ_TRY(launch_gather_rows(h, Xs, dc, d_idx, count, M, dBest));
  long long hidx[kMaxTopk];
  VZ_CUDA(cudaMemcpyAsync(hidx, d_idx, sizeof(long long) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(best_score, d_val, sizeof(double) * count, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaMemcpyAsync(best_x, dBest, sizeof(double) * (size_t)count * dc, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  if (best_index)
    for (int c = 0; c < count; ++c) best_index[c] = (hidx[c] == LLONG_MAX) ? -1 : (int64_t)hidx[c];
  return 0;
}

int vzgp_score_topk_pack(vzgp_handle* h, const double* Xs, const int32_t* Zs, int M, const vzgp_acq* acq,
                         int count, int64_t index_base, double* score_dev, double* payload_dev) {
  VZ_ARG(payload_dev != nullptr, "payload");
  VZ_ARG(M >= 1, "M >= 1");
  VZ_ARG(index_base >= 0 && index_base + (int64_t)M < (1LL << 53), "global indices must be exact in fp64");
  Guard g(h ? h->device : 0);
  const int dc = h ? h->dc : 0;
  double* dS = score_dev;
  if (!dS) {
    VZ_ARG(h != nullptr, "handle");
    VZ_TRY(h->out_dev.reserve(sizeof(double) * (size_t)M));
    dS = h->out_dev.as<double>();
  }
  VZ_TRY(check_scoring(h, Xs, Zs, M, acq, dS));
  VZ_ARG(h->dk == 0, "continuous features only");
  VZ_TRY(launch_score(h, Xs, Zs, M, acq, dS, nullptr, nullptr, nullptr, handle_acq(h)));
  long long* d_idx; double* d_val;
  VZ_TRY(topk_to_device(h, dS, M, count, &d_idx, &d_val));
  return launch_pack_topk(h, Xs, dc, d_idx, d_val, count, M, index_base, payload_dev);
}

int vzgp_merge_topk(vzgp_handle* h, const double* rows_dev, int n_rows, int width, int count,
                    double* out_dev, double* host_out) {
  VZ_ARG(h && rows_dev && out_dev, "handle / pointers");
  VZ_ARG(n_rows >= 1 && n_rows <= 2048, "1 <= n_rows <= 2048");
  VZ_ARG(width >= 2, "width >= 2");
  VZ_ARG(count >= 1 && count <= kMaxTopk, "1 <= count <= 256");
  Guard g(h->device);
  VZ_TRY(launch_merge_topk(h, rows_dev, n_rows, width, count, out_dev));
  if (host_out)
    VZ_CUDA(cudaMemcpyAsync(host_out, out_dev, sizeof(double) * (size_t)count * width, cudaMemcpyDeviceToHost, h->stream));
  return 0;
}

int vzgp_suggest_host(vzgp_handle* h, vzgp_exchange* x, int use_nccl, const double* Xs, int M, const vzgp_acq* acq,
                      int count, int64_t index_base, double* score_host, double* best_rows) {
  VZ_ARG(best_rows != nullptr, "best_rows");
  VZ_ARG(M >= 1, "M >= 1");
  VZ_ARG(index_base >= 0 && index_base + (int64_t)M < (1LL << 53), "global indices must be exact in fp64");
  static double dummy = 0.0;
  VZ_TRY(check_scoring(h, Xs, nullptr, M, acq, &dummy));
  VZ_ARG(h->dk == 0, "continuous features only");
  Guard g(h->device);
  const int dc = h->dc, w = dc + 2;
  VZ_ARG((size_t)2 * count * w * sizeof(double) <= kRowsBytes, "count * (Dc + 2) too large");
  double *dX, *o;
  VZ_TRY(score_host_enqueue(h, Xs, nullptr, M, acq, false, false, false, &dX, &o));
  long long* d_idx; double* d_val;
  VZ_TRY(topk_to_device(h, o, M, count, &d_idx, &d_val));
  double* payload = reinterpret_cast<double*>(h->small.as<char>() + kOffRows);   // [count][w], then the merged rows
  double* merged = payload + (size_t)count * w;
  VZ_TRY(launch_pack_topk(h, dX, dc, d_idx, d_val, count, M, index_base, payload));
  if (x != nullptr) {
    VZ_TRY(vzgp_allgather_topk(h, x, payload, merged, best_rows, use_nccl));
  } else {
    VZ_CUDA(cudaMemcpyAsync(best_rows, payload, sizeof(double) * (size_t)count * w, cudaMemcpyDeviceToHost, h->stream));
  }
  if (score_host) VZ_CUDA(cudaMemcpyAsync(score_host, o, sizeof(double) * (size_t)M, cudaMemcpyDeviceToHost, h->stream));
  VZ_CUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

}  // extern "C"
