// Times k_potf2_inv (64x64 diagonal-block Cholesky + inverse) in isolation: back-to-back launches
// with CUDA events, on a warmed-up GPU.  Build:
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/_bin/potf2_bench tools/potf2_bench.cu
#define VZ_POTF2_TIMING 1
#include "../vizier_b200/csrc/linalg.cu"
namespace vzgp {
void set_error(const char*, ...) {}
int raise_dyn_smem(const void* k, size_t b) { return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b) == cudaSuccess ? 0 : -2; }
}
#include <vector>
#include <cstdio>
__global__ void k_spin(double* x, int n) { double v = x[0]; for (int i = 0; i < n; ++i) v = fma(v, 1.0000001, 1e-9); x[0] = v; }
int main() {
  using namespace vzgp;
  const int ld = 64;
  std::vector<double> h(64 * 64);
  for (int i = 0; i < 64; ++i) for (int j = 0; j < 64; ++j) h[i * 64 + j] = (i == j ? 65.0 : 1.0 / (1 + abs(i - j)));
  double *A, *L, *Li; int* flag; double* sp;
  cudaMalloc(&A, sizeof(double) * 4096); cudaMalloc(&L, sizeof(double) * 4096); cudaMalloc(&Li, sizeof(double) * 4096);
  cudaMalloc(&flag, 4); cudaMalloc(&sp, 8); cudaMemset(sp, 0, 8);
  cudaMemcpy(A, h.data(), sizeof(double) * 4096, cudaMemcpyHostToDevice);
  cudaFuncSetAttribute(k_potf2_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDiagSmem);
  // warm the whole GPU so clocks are up
  for (int i = 0; i < 20; ++i) k_spin<<<132 * 8, 256>>>(sp, 200000);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int reps = 500;
  cudaEventRecord(e0);
  for (int r = 0; r < reps; ++r) {
    cudaMemcpyAsync(L, A, sizeof(double) * 4096, cudaMemcpyDeviceToDevice);
    k_potf2_inv<<<1, 256, kDiagSmem>>>(L, ld, 0, Li, ld, flag);
  }
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  cudaEventRecord(e0);
  for (int r = 0; r < reps; ++r) cudaMemcpyAsync(L, A, sizeof(double) * 4096, cudaMemcpyDeviceToDevice);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms2; cudaEventElapsedTime(&ms2, e0, e1);
  printf("{\"potf2_inv_us\": %.2f, \"copy_only_us\": %.2f, \"err\": \"%s\"}\n", 1e3 * ms / reps, 1e3 * ms2 / reps,
         cudaGetErrorString(cudaGetLastError()));
  long long ts[32];
  cudaMemcpyFromSymbol(ts, g_potf2_t, sizeof(ts));
  printf("phase cycles:");
  for (int i = 1; i <= 18; ++i) printf(" %d:%lld", i, ts[i] - ts[i - 1]);
  printf("  total %lld\n", ts[18] - ts[0]);
  return 0;
}
