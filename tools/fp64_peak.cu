// Measures the achievable FP64 throughput of this GPU: DFMA (vector pipe) and DMMA
// (mma.sync m8n8k4 / m16n8k8 / m16n8k16 f64) alone and together.  The result is the roofline
// denominator for the posterior-variance contraction (MEASURED_PEAKS.json has no fp64 entry).
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/_bin/fp64_peak tools/fp64_peak.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__global__ void k_dfma(double* out, int iters, double a, double b) {
  double c[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) c[i] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i] = fma(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += c[i];
  if (s == 123.456) out[0] = s;
}

__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__global__ void k_dmma884(double* out, int iters, double a, double b) {
  double c[8][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) { c[i][0] = i; c[i][1] = threadIdx.x; }
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dmma884(c[i][0], c[i][1], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  if (s == 123.456) out[0] = s;
}

__device__ __forceinline__ void dmma1688(double (&d)[4], const double (&a)[4], const double (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__global__ void k_dmma1688(double* out, int iters, double av, double bv) {
  double c[4][4];
  double a[4] = {av, av + 1, av + 2, av + 3}, b[2] = {bv, bv + 1};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[i][j] = i + j + threadIdx.x;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 4; ++i) dmma1688(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) s += c[i][j];
  if (s == 123.456) out[0] = s;
}

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}
__global__ void k_dmma16816(double* out, int iters, double av, double bv) {
  double c[4][4];
  double a[8], b[4];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = av + i;
#pragma unroll
  for (int i = 0; i < 4; ++i) b[i] = bv + i;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[i][j] = i + j + threadIdx.x;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 4; ++i) dmma16816(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) s += c[i][j];
  if (s == 123.456) out[0] = s;
}

// DFMA and DMMA interleaved in the same warp
__global__ void k_mixed(double* out, int iters, double a, double b) {
  double c[8][2], f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { c[i][0] = i; c[i][1] = threadIdx.x; f[i] = i * 0.5; }
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { dmma884(c[i][0], c[i][1], a, b); f[i] = fma(f[i], a, b); f[i] = fma(f[i], a, b); }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1] + f[i];
  if (s == 123.456) out[0] = s;
}

template <typename F>
static double time_ms(F launch, int reps) {
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  launch(); launch();
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(e0));
    launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  double* out; CK(cudaMalloc(&out, 8));
  const int sms = p.multiProcessorCount, ctas = sms * 8, threads = 256, iters = 4096;
  const double warps = (double)ctas * threads / 32;
  printf("{\"gpu\": \"%s\", \"sms\": %d", p.name, sms);
  double ms;
  ms = time_ms([&] { k_dfma<<<ctas, threads>>>(out, iters, 1.0000001, 1e-9); }, 5);
  printf(", \"dfma_tflops\": %.2f", 2.0 * 16 * iters * ctas * threads / ms * 1e-9);
  ms = time_ms([&] { k_dmma884<<<ctas, threads>>>(out, iters, 1.0000001, 1e-9); }, 5);
  printf(", \"dmma_m8n8k4_tflops\": %.2f", 2.0 * 8 * 8 * 4 * 8 * iters * warps / ms * 1e-9);
  ms = time_ms([&] { k_dmma1688<<<ctas, threads>>>(out, iters, 1.0000001, 1e-9); }, 5);
  printf(", \"dmma_m16n8k8_tflops\": %.2f", 2.0 * 16 * 8 * 8 * 4 * iters * warps / ms * 1e-9);
  ms = time_ms([&] { k_dmma16816<<<ctas, threads>>>(out, iters, 1.0000001, 1e-9); }, 5);
  printf(", \"dmma_m16n8k16_tflops\": %.2f", 2.0 * 16 * 8 * 16 * 4 * iters * warps / ms * 1e-9);
  ms = time_ms([&] { k_mixed<<<ctas, threads>>>(out, iters, 1.0000001, 1e-9); }, 5);
  printf(", \"mixed_dmma884_plus_2dfma_tflops\": %.2f", (2.0 * 256 * 8 * warps + 2.0 * 16 * ctas * threads) * iters / ms * 1e-9);
  printf("}\n");
  return 0;
}
