// Device-side building blocks: Matern-5/2, Philox4x32-10, and the fp64
// register-tiled GEMM main loop every dense kernel in this library is built on.
#pragma once

#include "common.cuh"

namespace vzgp {

// ---------------------------------------------------------------------------
// Matern-5/2 from the scaled squared distance (SURVEY A.1):
//   k = sf2*(1+s+s^2/3)*exp(-s),  s = sqrt(5*d2);   E = dk/d(d2) = -(5/6)*sf2*(1+s)*exp(-s)
// ---------------------------------------------------------------------------
__device__ __forceinline__ double matern52(double d2, double sf2) {
  double s = sqrt(5.0 * d2);
  return sf2 * (1.0 + s + s * s * (1.0 / 3.0)) * exp(-s);
}

__device__ __forceinline__ void matern52_with_grad(double d2, double sf2, double& k, double& e) {
  double s = sqrt(5.0 * d2);
  double es = exp(-s);
  k = sf2 * (1.0 + s + s * s * (1.0 / 3.0)) * es;
  e = -(5.0 / 6.0) * sf2 * (1.0 + s) * es;
}

// ---------------------------------------------------------------------------
// Philox4x32-10; bit-identical to oracle/eagle_oracle.py::philox4x32.
// ---------------------------------------------------------------------------
constexpr uint32_t kStreamInitPool = 0;
constexpr uint32_t kStreamPerturbSign = 1;
constexpr uint32_t kStreamTrim = 2;
constexpr uint32_t kStreamRandomPool = 3;

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t& o0,
                                              uint32_t& o1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  o0 = c0; o1 = c1;
}

// Uniform double in [0,1) for (seed, stream, iteration, element); element is 32-bit
// in counter word 0 and its high part (pools > 2^32 elements) goes to word 3.
__device__ __forceinline__ double philox_uniform(uint64_t seed, uint32_t stream, uint32_t iteration,
                                                 uint64_t element) {
  uint32_t w0, w1;
  philox4x32_10(static_cast<uint32_t>(element), iteration, stream,
                static_cast<uint32_t>(element >> 32), static_cast<uint32_t>(seed),
                static_cast<uint32_t>(seed >> 32), w0, w1);
  return (static_cast<double>(w0 >> 5) * 67108864.0 + static_cast<double>(w1 >> 6)) *
         (1.0 / 9007199254740992.0);
}

// ---------------------------------------------------------------------------
// fp64 GEMM main loop.
//
// acc[i][j] += sum_{k in [kbegin,kend)} A(m0 + tm(i), k) * B(n0 + tn(j), k)
//
// Operand element (row, k) lives at ptr[row*ld + k] when *_KMAJOR is false
// (k contiguous: "row-major [row,k]") and at ptr[k*ld + row] when true (row
// contiguous).  BM x BN CTA tile, BK k-slab, TTM x TTN register tile per
// thread, (BM/TTM)*(BN/TTN) threads.  Slabs are staged k-major in shared
// memory ([BK][BM+PAD]) so each thread reads its TTM (TTN) consecutive rows
// with 16-byte loads; global->shared goes through registers so the next slab
// is in flight while the current one is multiplied (double-buffered smem, one
// __syncthreads per slab).  All extents are multiples of the tile sizes (the
// library pads every matrix to 64), all pointers 16-byte aligned.
// Thread (ty, tx) = (tid / (BN/TTN), tid % (BN/TTN)).  Its register tile is made of
// 2-wide chunks strided across the CTA tile so that the 16-byte shared-memory
// reads of neighbouring lanes are contiguous (no bank conflicts) and global
// stores of a row are coalesced:  row_of(ty,i) / col_of(tx,j) below.
// ---------------------------------------------------------------------------
template <int BM, int BN, int BK, int TTM, int TTN>
struct GemmCfg {
  static constexpr int kThreads = (BM / TTM) * (BN / TTN);
  static constexpr int kPad = 2;
  static constexpr int kLdA = BM + kPad;
  static constexpr int kLdB = BN + kPad;
  static constexpr int kSmemDoubles = 2 * BK * (kLdA + kLdB);
  static constexpr size_t kSmemBytes = sizeof(double) * kSmemDoubles;
  static_assert((BM * BK) % (2 * kThreads) == 0, "A slab must split into double2 per thread");
  static_assert((BN * BK) % (2 * kThreads) == 0, "B slab must split into double2 per thread");
  static_assert(TTM % 2 == 0 && TTN % 2 == 0, "register tile must be even");
  static constexpr int kRowChunk = BM / (TTM / 2);  // stride between a thread's row pairs
  static constexpr int kColChunk = BN / (TTN / 2);
  __host__ __device__ static constexpr int row_of(int ty, int i) {
    return (i / 2) * kRowChunk + ty * 2 + (i % 2);
  }
  __host__ __device__ static constexpr int col_of(int tx, int j) {
    return (j / 2) * kColChunk + tx * 2 + (j % 2);
  }
};

template <int ROWS, int BK, int THREADS, bool KMAJOR>
struct SlabLoader {
  static constexpr int kVec = ROWS * BK / (2 * THREADS);  // double2 loads per thread
  double2 v[kVec];

  __device__ __forceinline__ void load(const double* __restrict__ p, int ld, int row0, int k0,
                                       int tid) {
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      int e = (i * THREADS + tid) * 2;
      if (KMAJOR) {
        int k = e / ROWS, r = e % ROWS;
        v[i] = __ldcg(reinterpret_cast<const double2*>(p + (size_t)(k0 + k) * ld + row0 + r));
      } else {
        int r = e / BK, k = e % BK;
        v[i] = __ldcg(reinterpret_cast<const double2*>(p + (size_t)(row0 + r) * ld + k0 + k));
      }
    }
  }
  __device__ __forceinline__ void store(double* s, int lds, int tid) const {
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      int e = (i * THREADS + tid) * 2;
      if (KMAJOR) {
        int k = e / ROWS, r = e % ROWS;
        *reinterpret_cast<double2*>(s + k * lds + r) = v[i];
      } else {
        int r = e / BK, k = e % BK;
        s[k * lds + r] = v[i].x;
        s[(k + 1) * lds + r] = v[i].y;
      }
    }
  }
};

template <int BM, int BN, int BK, int TTM, int TTN, bool A_KMAJOR, bool B_KMAJOR>
__device__ __forceinline__ void gemm_mainloop(const double* __restrict__ A, int lda, int m0,
                                              const double* __restrict__ B, int ldb, int n0,
                                              int kbegin, int kend, double (&acc)[TTM][TTN],
                                              double* smem) {
  using Cfg = GemmCfg<BM, BN, BK, TTM, TTN>;
  constexpr int T = Cfg::kThreads;
  const int tid = threadIdx.x;
  const int ty = tid / (BN / TTN), tx = tid % (BN / TTN);
  double* As = smem;                           // [2][BK][kLdA]
  double* Bs = smem + 2 * BK * Cfg::kLdA;      // [2][BK][kLdB]
  SlabLoader<BM, BK, T, A_KMAJOR> la;
  SlabLoader<BN, BK, T, B_KMAJOR> lb;

  if (kbegin >= kend) return;
  la.load(A, lda, m0, kbegin, tid);
  lb.load(B, ldb, n0, kbegin, tid);
  la.store(As, Cfg::kLdA, tid);
  lb.store(Bs, Cfg::kLdB, tid);
  __syncthreads();
  int buf = 0;
  for (int k0 = kbegin; k0 < kend; k0 += BK) {
    const bool more = (k0 + BK) < kend;
    if (more) {
      la.load(A, lda, m0, k0 + BK, tid);
      lb.load(B, ldb, n0, k0 + BK, tid);
    }
    const double* as = As + buf * BK * Cfg::kLdA + ty * 2;
    const double* bs = Bs + buf * BK * Cfg::kLdB + tx * 2;
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      double a[TTM], b[TTN];
#pragma unroll
      for (int i = 0; i < TTM; i += 2) {
        double2 t =
            *reinterpret_cast<const double2*>(as + kk * Cfg::kLdA + (i / 2) * Cfg::kRowChunk);
        a[i] = t.x; a[i + 1] = t.y;
      }
#pragma unroll
      for (int j = 0; j < TTN; j += 2) {
        double2 t =
            *reinterpret_cast<const double2*>(bs + kk * Cfg::kLdB + (j / 2) * Cfg::kColChunk);
        b[j] = t.x; b[j + 1] = t.y;
      }
#pragma unroll
      for (int i = 0; i < TTM; ++i)
#pragma unroll
        for (int j = 0; j < TTN; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
    if (more) {
      la.store(As + (buf ^ 1) * BK * Cfg::kLdA, Cfg::kLdA, tid);
      lb.store(Bs + (buf ^ 1) * BK * Cfg::kLdB, Cfg::kLdB, tid);
    }
    __syncthreads();
    buf ^= 1;
  }
}

// Block-wide sum of one double per thread (result valid in thread 0).  red: >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    v = lane < nw ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  }
  return v;
}

// D(8x8) += A(8x4, row) * B(4x8, col); lane l holds A[l/4][l%4], B[k=l%4][n=l/4],
// D[l/4][2*(l%4)+{0,1}]  (PTX ISA, mma.m8n8k4 .f64 fragment layout).
__device__ __forceinline__ void dmma_8x8x4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

// D[16x8] += A[16x8] B[8x8] (mma.sync m16n8k8 f64, sm_90).  Lane (g = lane/4, t = lane%4): a0 = A[g][t],
// a1 = A[g+8][t], a2 = A[g][t+4], a3 = A[g+8][t+4]; b0 = B[t][g], b1 = B[t+4][g]; d0, d1 = D[g][2t, 2t+1],
// d2, d3 = D[g+8][2t, 2t+1].
__device__ __forceinline__ void dmma_16x8x8(double& d0, double& d1, double& d2, double& d3, double a0, double a1, double a2,
                                            double a3, double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
               : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}

// m16n8k4 f64 (sm_90): A 16 x 4 (a0 row g, a1 row g + 8, column t), B 4 x 8 (b0 row t, column g).
__device__ __forceinline__ void dmma_16x8x4(double& d0, double& d1, double& d2, double& d3, double a0, double a1, double b0) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
               : "d"(a0), "d"(a1), "d"(b0));
}

}  // namespace vzgp
