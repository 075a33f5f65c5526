// Building blocks shared by K8 (nmf.cu) and K9 (puresvd.cu): a deterministic warp-per-row CSR x tall SpMM with up to
// F_MAX columns, and the fp64 Gram M^T M of a tall fp32 matrix with its split partials summed in a fixed order.  Both
// accumulate in fp64.  The kernels are static so that each translation unit that includes this header has its own copy.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace b200 {
namespace nmf {

constexpr int KMAX = 16;  // columns per lane in the warp-per-row kernels
constexpr int F_MAX = 32 * KMAX;
constexpr int WARPS = 8;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// out[r, :] = sum over (j, x) in row r of (ptr, idx, val):  x * M[j, :]
static __global__ void __launch_bounds__(256) spmm_kernel(int n_rows, const int* __restrict__ ptr, const int* __restrict__ idx,
                                                          const float* __restrict__ val, const float* __restrict__ M, int f,
                                                          float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  double acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = 0.0;
  const int s = ptr[row], e = ptr[row + 1];
  for (int q0 = s; q0 < e; q0 += 32) {
    int jj = 0;
    float xx = 0.f;
    if (q0 + lane < e) { jj = idx[q0 + lane]; xx = val[q0 + lane]; }
    const int cnt = min(32, e - q0);
    for (int t = 0; t < cnt; ++t) {
      const int j = __shfl_sync(0xffffffffu, jj, t);
      const double x = __shfl_sync(0xffffffffu, xx, t);
      const float* m = M + (size_t)j * f;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const int c = lane + 32 * k;
        if (c < f) acc[k] += x * (double)m[c];
      }
    }
  }
  float* o = out + (size_t)row * f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    const int c = lane + 32 * k;
    if (c < f) o[c] = (float)acc[k];
  }
}

// P[split][a][b] = sum over the split's rows i of M[i, a] M[i, b]; blockIdx.x = output tile, blockIdx.y = split
static __global__ void __launch_bounds__(256) gram_partial_kernel(int n, int f, const float* __restrict__ M, int rows_per_split,
                                                                  double* __restrict__ P) {
  __shared__ float Ma[32][33], Mb[32][33];
  const int tiles = (f + 31) / 32;
  const int ta = blockIdx.x / tiles, tb = blockIdx.x % tiles;
  const int ty = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r_begin = blockIdx.y * rows_per_split, r_end = min(n, r_begin + rows_per_split);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int r0 = r_begin; r0 < r_end; r0 += 32) {
    for (int e = threadIdx.x; e < 1024; e += 256) {
      const int rr = e >> 5, cc = e & 31, row = r0 + rr;
      const bool in = row < r_end;
      Ma[rr][cc] = in && ta * 32 + cc < f ? M[(size_t)row * f + ta * 32 + cc] : 0.f;
      Mb[rr][cc] = in && tb * 32 + cc < f ? M[(size_t)row * f + tb * 32 + cc] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr) {
      const double mb = Mb[rr][lane];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += (double)Ma[rr][ty + 8 * j] * mb;
    }
    __syncthreads();
  }
  const int b = tb * 32 + lane;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int a = ta * 32 + ty + 8 * j;
    if (a < f && b < f) P[(size_t)blockIdx.y * f * f + (size_t)a * f + b] = acc[j];
  }
}

// out[e] = sum over s < n_splits of P[s * len + e], in split order
static __global__ void sum_splits_kernel(const double* __restrict__ P, int n_splits, long long len, double* __restrict__ out) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= len) return;
  double s = 0.0;
  for (int k = 0; k < n_splits; ++k) s += P[(size_t)k * len + e];
  out[e] = s;
}

// rows per split of the fp64 split reductions: about 4 CTAs per SM in all, at least 32 rows per split
inline int split_rows(int n, int blocks_per_split) {
  const int want = std::max(1, (4 * sm_count() + blocks_per_split - 1) / blocks_per_split);
  const int per = (int)div_up(div_up(n, want), 32) * 32;
  return std::max(per, 32);
}

// the split count of an n-row reduction; not monotonic in n (the rows per split go up in steps of 32)
inline int n_splits(int n, int blocks_per_split) { return (int)div_up(n, split_rows(n, blocks_per_split)); }

}  // namespace nmf
}  // namespace b200
