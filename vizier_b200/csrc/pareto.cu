// Pareto dominance, Pareto rank and the randomized cumulative hypervolume from the origin of a set of FP64 points
// (xla_pareto.py / hypervolume.py of the reference).  DESIGN.md §6n.
//
// Dominance ("a dominates p": all(p <= a), and when strict also any(a > p)) is pure comparison, so the outputs are
// exact; a NaN coordinate makes p <= a false, so a row with a NaN neither dominates nor is dominated.  The hypervolume
// sums its per-vector terms in a fixed order (per CTA, then across CTAs in a second kernel), so repeated calls are
// bit-identical.
#include <algorithm>

#include "launchers.h"

namespace vzgp {
namespace {

constexpr int kDomThreads = 256;       // one point per thread
constexpr int kSlabDoubles = 4096;     // 32 KiB of `against` rows staged in shared memory at a time
constexpr int kRowUnroll = 8;          // rows compared between two checks of the frontier's early exit
constexpr int kHvThreads = 256;        // one point of the chunk per thread
constexpr int kHvGroup = 8;            // vectors scanned per round (one barrier per round)
constexpr int kHvWarps = kHvThreads / 32;
constexpr size_t kHvMaxScratch = size_t(256) << 20;   // per-CTA partial sums [ctas][n], kept by the handle

// Rows of `against` are staged as [rows][kM] (kM = m rounded up to a power of two); the padded coordinates are 0 in the
// point and in the row, which keeps p <= a true and a > p false, so they change nothing.  kRank = false: optimal[i] is
// cleared when a row dominates point i, and a CTA stops once all its points are dominated.  kRank = true: rank[i] gains
// the number of rows that dominate point i.  blockIdx.y selects the CTA's range of `against` rows.
template <int kM, bool kRank>
__global__ void __launch_bounds__(kDomThreads) k_pareto_dominance(const double* __restrict__ pts, int n,
                                                                   const double* __restrict__ against, int n_against,
                                                                   int m, int strict, int rows_per_cta,
                                                                   uint8_t* __restrict__ optimal,
                                                                   int* __restrict__ rank) {
  constexpr int kRows = kSlabDoubles / kM;
  __shared__ double slab[kSlabDoubles];
  const int i = blockIdx.x * kDomThreads + threadIdx.x;
  double p[kM];
#pragma unroll
  for (int k = 0; k < kM; ++k) p[k] = (i < n && k < m) ? pts[(size_t)i * m + k] : 0.0;
  const int begin = blockIdx.y * rows_per_cta;
  const int end = min(n_against, begin + rows_per_cta);
  bool dominated = i >= n;   // points past n take no part in the CTA's vote
  int count = 0;
  for (int s = begin; s < end; s += kRows) {
    // the barrier before the slab is overwritten doubles as the CTA's vote: stop when every point is dominated
    if (kRank) {
      __syncthreads();
    } else if (__syncthreads_and(dominated)) {
      break;
    }
    const int rows = min(kRows, end - s);
    // rows past the range are NaN: p <= NaN is false, so they dominate nothing
    const int rows_padded = (rows + kRowUnroll - 1) / kRowUnroll * kRowUnroll;
    for (int e = threadIdx.x; e < rows_padded * kM; e += kDomThreads) {
      const int r = e / kM, k = e % kM;
      slab[e] = r >= rows ? __longlong_as_double(0x7ff8000000000000LL)
                          : (k < m ? against[(size_t)(s + r) * m + k] : 0.0);
    }
    __syncthreads();
    if (kRank || !dominated) {
      for (int r0 = 0; r0 < rows_padded; r0 += kRowUnroll) {
        bool any = false;
#pragma unroll
        for (int r = r0; r < r0 + kRowUnroll; ++r) {
          const double* a = slab + r * kM;
          bool le = true, gt = false;
#pragma unroll
          for (int k = 0; k < kM; ++k) {
            le &= p[k] <= a[k];
            gt |= a[k] > p[k];
          }
          const bool dom = le && (gt || !strict);
          count += dom ? 1 : 0;
          any |= dom;
        }
        if (!kRank && any) {
          dominated = true;
          break;
        }
      }
    }
  }
  if (i < n) {
    if (kRank) {
      if (count) atomicAdd(rank + i, count);
    } else if (dominated) {
      optimal[i] = 0;
    }
  }
}

// NumPy's minimum / maximum: NaN if either operand is NaN.
__device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ double int_pow(double x, int e) {
  double r = 1.0;
  for (;;) {
    if (e & 1) r *= x;
    e >>= 1;
    if (!e) return r;
    x *= x;
  }
}

// CTA b owns vectors [b * vpc, b * vpc + nv).  Points are taken in chunks of kHvThreads (thread t <-> point c0 + t):
// for kHvGroup vectors at a time each thread forms min_k p[j,k] / v[k], the CTA max-scans that along the chunk (warp
// shuffles, then the warp totals and the running max carried from the previous chunk), and each thread adds
// (scanned value)^m to its point's sum, vectors in ascending order.  partial[b][j] = that sum.
__global__ void __launch_bounds__(kHvThreads) k_cum_hypervolume(const double* __restrict__ pts, int n, int m,
                                                                const double* __restrict__ vec, int v_total, int vpc,
                                                                double* __restrict__ partial) {
  extern __shared__ double sh[];
  double* sp = sh;                                   // [m][kHvThreads] the chunk's points, coordinate-major
  double* carry = sp + (size_t)m * kHvThreads;       // [2][vpc] running max per vector, by chunk parity
  double* wt = carry + 2 * (size_t)vpc;              // [2][kHvGroup][kHvWarps] warp totals, by round parity
  const int v0 = blockIdx.x * vpc;
  const int nv = min(vpc, v_total - v0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int e = threadIdx.x; e < nv; e += kHvThreads) carry[e] = -INFINITY;
  int par = 0;
  for (int c0 = 0, chunk = 0; c0 < n; c0 += kHvThreads, ++chunk) {
    const int j = c0 + threadIdx.x;
    const int rows = min(kHvThreads, n - c0);
    __syncthreads();   // the previous chunk's reads of sp are done
    for (int e = threadIdx.x; e < rows * m; e += kHvThreads) {
      const int r = e / m;
      sp[(e - r * m) * kHvThreads + r] = pts[(size_t)c0 * m + e];
    }
    __syncthreads();
    const double* cin = carry + (chunk & 1) * vpc;
    double* cout = carry + ((chunk + 1) & 1) * vpc;
    double acc = 0.0;
    for (int g0 = 0; g0 < nv; g0 += kHvGroup) {
      double r[kHvGroup];
#pragma unroll
      for (int g = 0; g < kHvGroup; ++g) r[g] = j < n ? INFINITY : -INFINITY;   // points past n end the scan
      if (j < n) {
        for (int k = 0; k < m; ++k) {
          const double x = sp[k * kHvThreads + threadIdx.x];
#pragma unroll
          for (int g = 0; g < kHvGroup; ++g) {
            const int v = v0 + min(g0 + g, nv - 1);   // rounds past nv repeat the last vector; their terms are dropped
            r[g] = nan_min(r[g], x / __ldg(vec + (size_t)v * m + k));
          }
        }
      }
#pragma unroll
      for (int g = 0; g < kHvGroup; ++g) {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double t = __shfl_up_sync(0xffffffffu, r[g], o);
          if (lane >= o) r[g] = nan_max(r[g], t);
        }
      }
      double* w = wt + par * (kHvGroup * kHvWarps);
      if (lane == 31) {
#pragma unroll
        for (int g = 0; g < kHvGroup; ++g) w[g * kHvWarps + warp] = r[g];
      }
      __syncthreads();   // wt is double-buffered, so the next round's writes need no second barrier
#pragma unroll
      for (int g = 0; g < kHvGroup; ++g) {
        if (g0 + g < nv) {
          double pre = cin[g0 + g];
          for (int ww = 0; ww < warp; ++ww) pre = nan_max(pre, w[g * kHvWarps + ww]);
          const double val = nan_max(pre, r[g]);
          if (j < n) acc += int_pow(val, m);
          if (threadIdx.x == kHvThreads - 1) cout[g0 + g] = val;   // the running max through the whole chunk
        }
      }
      par ^= 1;
    }
    if (j < n) partial[(size_t)blockIdx.x * n + j] = acc;
  }
}

// out[j] = (sum over CTAs b, ascending, of partial[b][j]) / v_total.
__global__ void k_cum_hypervolume_reduce(const double* __restrict__ partial, int ctas, int n, int v_total,
                                         double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double s = 0.0;
  for (int b = 0; b < ctas; ++b) s += partial[(size_t)b * n + j];
  out[j] = s / (double)v_total;
}

template <int kM>
int launch_dominance_m(vzgp_handle* h, const double* pts, int n, const double* against, int n_against, int m,
                       int strict, uint8_t* optimal, int* rank) {
  constexpr int kRows = kSlabDoubles / kM;
  const int gx = (n + kDomThreads - 1) / kDomThreads;
  // split `against` between CTAs until the grid covers the SMs twice; each CTA's range is whole slabs
  const int slabs = (n_against + kRows - 1) / kRows;
  const int want = (2 * h->sm_count + gx - 1) / gx;
  const int gy = std::max(1, std::min(slabs, want));
  const int rows_per_cta = (slabs + gy - 1) / gy * kRows;
  const int gy_used = (n_against + rows_per_cta - 1) / rows_per_cta;
  const dim3 grid(gx, std::max(1, gy_used));
  if (rank) {
    k_pareto_dominance<kM, true><<<grid, kDomThreads, 0, h->stream>>>(pts, n, against, n_against, m, 1,
                                                                     rows_per_cta, nullptr, rank);
  } else {
    k_pareto_dominance<kM, false><<<grid, kDomThreads, 0, h->stream>>>(pts, n, against, n_against, m, strict,
                                                                      rows_per_cta, optimal, nullptr);
  }
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace

int launch_pareto_dominance(vzgp_handle* h, const double* pts, int n, const double* against, int n_against, int m,
                            int strict, uint8_t* optimal, int* rank) {
  if (rank) {
    VZ_CUDA(cudaMemsetAsync(rank, 0, sizeof(int) * (size_t)n, h->stream));
  } else {
    VZ_CUDA(cudaMemsetAsync(optimal, 1, (size_t)n, h->stream));
  }
  if (n_against == 0) return 0;
  if (m <= 1) return launch_dominance_m<1>(h, pts, n, against, n_against, m, strict, optimal, rank);
  if (m <= 2) return launch_dominance_m<2>(h, pts, n, against, n_against, m, strict, optimal, rank);
  if (m <= 4) return launch_dominance_m<4>(h, pts, n, against, n_against, m, strict, optimal, rank);
  if (m <= 8) return launch_dominance_m<8>(h, pts, n, against, n_against, m, strict, optimal, rank);
  if (m <= 16) return launch_dominance_m<16>(h, pts, n, against, n_against, m, strict, optimal, rank);
  if (m <= 32) return launch_dominance_m<32>(h, pts, n, against, n_against, m, strict, optimal, rank);
  return launch_dominance_m<kMaxParetoMetrics>(h, pts, n, against, n_against, m, strict, optimal, rank);
}

int launch_cum_hypervolume(vzgp_handle* h, const double* pts, int n, int m, const double* vec, int v, double* out) {
  // About four CTAs per SM, each a whole number of kHvGroup-vector rounds.  Fewer, wider CTAs when the partial sums
  // [CTAs][n] would pass kHvMaxScratch; a CTA's vectors are bounded by its running maxima in shared memory.
  const size_t fixed_smem = sizeof(double) * ((size_t)m * kHvThreads + 2 * kHvGroup * kHvWarps);
  const int64_t vpc_max = (int64_t)((kMaxDynSmem - fixed_smem) / (2 * sizeof(double))) / kHvGroup * kHvGroup;
  const int64_t ctas_max = (int64_t)(kHvMaxScratch / (sizeof(double) * (size_t)n));
  int64_t vpc = std::max(ceil_div64(v, 4 * (int64_t)h->sm_count), ctas_max > 0 ? ceil_div64(v, ctas_max) : v);
  vpc = ceil_div64(vpc, kHvGroup) * kHvGroup;
  VZ_ARG(ctas_max > 0 && vpc <= vpc_max,
         "n x ceil(v / vectors per CTA) partial sums must fit the 256 MiB hypervolume scratch");
  const int ctas = (int)ceil_div64(v, vpc);
  const size_t scratch = sizeof(double) * (size_t)ctas * (size_t)n;
  // A larger buffer replaces the old one, which earlier launches on the stream may still be reading.
  if (scratch > h->pareto.bytes && h->pareto.ptr) VZ_CUDA(cudaStreamSynchronize(h->stream));
  VZ_TRY(h->pareto.reserve(scratch));
  const size_t smem = fixed_smem + sizeof(double) * 2 * (size_t)vpc;
  VZ_TRY(raise_dyn_smem((const void*)k_cum_hypervolume, smem));
  double* partial = h->pareto.as<double>();
  k_cum_hypervolume<<<ctas, kHvThreads, smem, h->stream>>>(pts, n, m, vec, v, (int)vpc, partial);
  VZ_CHECK_LAUNCH();
  h->launches++;
  k_cum_hypervolume_reduce<<<(n + 255) / 256, 256, 0, h->stream>>>(partial, ctas, n, v, out);
  VZ_CHECK_LAUNCH();
  h->launches++;
  return 0;
}

}  // namespace vzgp
