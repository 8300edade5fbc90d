// potf2_inv_64 (round 1) against potf2_inv_64_la (look-ahead, round 2) in isolation: one CTA of 256 threads
// factors + inverts the same 64 x 64 SPD block REPS times from shared memory; cycles per call from clock64
// around the whole loop (no stamps inside the routines), results compared with each other.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -maxrregcount=96 -o tools/_bin/potf2_la_bench tools/potf2_la_bench.cu
#include <cstdio>
#include <vector>
#include "../vizier_b200/csrc/potf2.cuh"
#include "../vizier_b200/csrc/potf2_la.cuh"
namespace vzgp { void set_error(const char*, ...) {} }
using namespace vzgp;
constexpr int REPS = 200;
template <int WHICH>
__global__ void __launch_bounds__(256) k_bench(const double* __restrict__ A, double* __restrict__ L, double* __restrict__ X,
                                               long long* cyc) {
  extern __shared__ double smem[];
  constexpr int LD = 66;
  double* a = smem; double* x = a + 64 * LD; double* t = x + 64 * LD;
  __shared__ double rd[64];
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  long long total = 0;
  for (int rep = 0; rep < REPS; ++rep) {
    for (int e = tid; e < 4096; e += 256) {
      const int i = e >> 6, j = e & 63;
      a[i * LD + j] = ((j >> 4) > (i >> 4)) ? 0.0 : A[e];
      x[i * LD + j] = 0.0;
    }
    if (tid == 0) s_bad = 0;
    __syncthreads();
    const long long t0 = clock64();
    if (WHICH == 0) potf2_inv_64(a, x, t, rd, &s_bad); else potf2_inv_64_la(a, x, t, rd, &s_bad);
    const long long t1 = clock64();
    total += t1 - t0;
    __syncthreads();
  }
  if (tid == 0) cyc[WHICH] = total / REPS;
  for (int e = tid; e < 4096; e += 256) { L[e] = a[(e >> 6) * LD + (e & 63)]; X[e] = x[(e >> 6) * LD + (e & 63)]; }
}
int main() {
  std::vector<double> h(4096), l0(4096), x0(4096), l1(4096), x1(4096);
  for (int i = 0; i < 64; ++i) for (int j = 0; j < 64; ++j) h[i * 64 + j] = (i == j ? 3.0 : 1.0 / (1 + abs(i - j)));
  double *A, *L, *X; long long* cyc;
  cudaMalloc(&A, 8 * 4096); cudaMalloc(&L, 8 * 4096); cudaMalloc(&X, 8 * 4096); cudaMalloc(&cyc, 16);
  cudaMemcpy(A, h.data(), 8 * 4096, cudaMemcpyHostToDevice);
  const size_t sm = sizeof(double) * (2 * 64 * 66 + 32 * 34);
  cudaFuncSetAttribute(k_bench<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
  cudaFuncSetAttribute(k_bench<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
  for (int w = 0; w < 3; ++w) {
    k_bench<0><<<1, 256, sm>>>(A, L, X, cyc);
    cudaMemcpy(l0.data(), L, 8 * 4096, cudaMemcpyDeviceToHost); cudaMemcpy(x0.data(), X, 8 * 4096, cudaMemcpyDeviceToHost);
    k_bench<1><<<1, 256, sm>>>(A, L, X, cyc);
    cudaMemcpy(l1.data(), L, 8 * 4096, cudaMemcpyDeviceToHost); cudaMemcpy(x1.data(), X, 8 * 4096, cudaMemcpyDeviceToHost);
  }
  long long c[2]; cudaMemcpy(c, cyc, 16, cudaMemcpyDeviceToHost);
  double dl = 0, dx = 0;
  for (int e = 0; e < 4096; ++e) { dl = fmax(dl, fabs(l0[e] - l1[e])); dx = fmax(dx, fabs(x0[e] - x1[e])); }
  // residual of the look-ahead result: L L^T - A and X L - I
  double r1 = 0, r2 = 0;
  for (int i = 0; i < 64; ++i) for (int j = 0; j <= i; ++j) {
    double s = 0, u = 0;
    for (int k = 0; k < 64; ++k) { s += l1[i * 64 + k] * l1[j * 64 + k]; u += x1[i * 64 + k] * l1[k * 64 + j]; }
    r1 = fmax(r1, fabs(s - h[i * 64 + j])); r2 = fmax(r2, fabs(u - (i == j ? 1.0 : 0.0)));
  }
  printf("{\"potf2_inv_64_cycles\": %lld, \"potf2_inv_64_la_cycles\": %lld, \"max_dL\": %.3e, \"max_dX\": %.3e, \"res_LLt\": %.3e, \"res_XL\": %.3e, \"err\": \"%s\"}\n",
         c[0], c[1], dl, dx, r1, r2, cudaGetErrorString(cudaGetLastError()));
  return 0;
}
