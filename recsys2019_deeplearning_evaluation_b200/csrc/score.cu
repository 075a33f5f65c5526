// K6: batch scoring behind _compute_item_score / recommend, sm_90a.
//
// Replaces
//   Base/BaseSimilarityMatrixRecommender.py:73-92   item scores = URM[users] . W_sparse           (SpMM -> dense block)
//   Base/BaseSimilarityMatrixRecommender.py:97-116  user-based twin  W_sparse[users] . URM
//   Base/BaseMatrixFactorizationRecommender.py:38-70 scores = U[users] . V^T (+ biases)
//   Base/BaseRecommender.py:164-196                 seen items -> -inf, per-row top-`cutoff`
// Outputs are dense [B, n_items] fp32 blocks (the Evaluator asks for B <= 1000 users at a time,
// Base/Evaluation/Evaluator.py:422).  Roofline: HBM, dominated by the B*n_items*4 bytes written (+ read back by the
// mask / top-N passes) and, for the sparse product, 8 bytes per gathered (j, w) pair of W.
#include <algorithm>

#include "common.cuh"

namespace b200 {
namespace score {

typedef unsigned long long u64;

// out[b, :] = sum over (i, r) in row users[b] of A:  r * Brow(i)   -- A, B both CSR; one CTA per output row
__global__ void __launch_bounds__(512) spmm_rows_kernel(const int* __restrict__ users, int n_users_block,
                                                        const int* __restrict__ a_ptr, const int* __restrict__ a_idx,
                                                        const float* __restrict__ a_val, const int* __restrict__ b_ptr,
                                                        const int* __restrict__ b_idx, const float* __restrict__ b_val,
                                                        int n_out_cols, float* out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  for (int b = blockIdx.x; b < n_users_block; b += gridDim.x) {
    float* o = out + (size_t)b * n_out_cols;
    for (int j = tid; j < n_out_cols; j += blockDim.x) o[j] = 0.f;
    __syncthreads();
    const int u = users[b];
    const int s = a_ptr[u], e = a_ptr[u + 1];
    for (int k = s + warp; k < e; k += nwarps) {
      const int i = a_idx[k];
      const float r = a_val[k];
      if (b_ptr) {
        for (int q = b_ptr[i] + lane; q < b_ptr[i + 1]; q += 32) atomicAdd(o + b_idx[q], r * b_val[q]);
      } else {  // dense B: row i is b_val[i * n_out_cols ..]
        const float* brow = b_val + (size_t)i * n_out_cols;
        for (int j = lane; j < n_out_cols; j += 32) atomicAdd(o + j, r * brow[j]);
      }
    }
    __syncthreads();
  }
}

// out[b, j] = U[users[b], :] . VT[:, j] (+ mu + bu[users[b]] + bi[j]);  VT is the transposed item-factor matrix
// [f, n_items] so that consecutive threads read consecutive items.  8 users per thread share every VT load.
constexpr int UT = 8;
__global__ void __launch_bounds__(256) mf_scores_kernel(const int* __restrict__ users, int n_users_block,
                                                        const float* __restrict__ U, const float* __restrict__ VT, int f,
                                                        int n_items, const float* __restrict__ bu, const float* __restrict__ bi,
                                                        const float* __restrict__ mu, float* out) {
  extern __shared__ float ush[];  // [UT][f]
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b0 = blockIdx.y * UT;
  for (int t = threadIdx.x; t < UT * f; t += blockDim.x) {
    const int bb = b0 + t / f;
    ush[t] = bb < n_users_block ? U[(size_t)users[bb] * f + (t % f)] : 0.f;
  }
  __syncthreads();
  if (j >= n_items) return;
  float acc[UT];
#pragma unroll
  for (int k = 0; k < UT; ++k) acc[k] = 0.f;
  for (int q = 0; q < f; ++q) {
    const float v = VT[(size_t)q * n_items + j];
#pragma unroll
    for (int k = 0; k < UT; ++k) acc[k] += ush[k * f + q] * v;
  }
  const float base = mu ? mu[0] + bi[j] : 0.f;
#pragma unroll
  for (int k = 0; k < UT; ++k) {
    const int bb = b0 + k;
    if (bb < n_users_block) out[(size_t)bb * n_items + j] = acc[k] + base + (mu ? bu[users[bb]] : 0.f);
  }
}

__global__ void transpose_kernel(const float* __restrict__ in, int rows, int cols, float* out) {
  __shared__ float tile[32][33];
  const int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
  for (int k = threadIdx.y; k < 32; k += blockDim.y)
    if (x < cols && y0 + k < rows) tile[k][threadIdx.x] = in[(size_t)(y0 + k) * cols + x];
  __syncthreads();
  const int ox = blockIdx.y * 32 + threadIdx.x, oy0 = blockIdx.x * 32;
  for (int k = threadIdx.y; k < 32; k += blockDim.y)
    if (ox < rows && oy0 + k < cols) out[(size_t)(oy0 + k) * rows + ox] = tile[threadIdx.x][k];
}

// scores[b, seen items of users[b]] = -inf (BaseRecommender.py:164-169); one warp per user
__global__ void mask_seen_kernel(const int* __restrict__ users, int n_users_block, const int* __restrict__ ptr,
                                 const int* __restrict__ idx, int n_items, float* scores) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_users_block) return;
  const int u = users[warp];
  for (int k = ptr[u] + lane; k < ptr[u + 1]; k += 32) scores[(size_t)warp * n_items + idx[k]] = -INFINITY;
}

// items_to_compute (BaseSimilarityMatrixRecommender.py:80-86): every other item -> -inf.  keep[j] != 0 marks kept items.
__global__ void mask_items_kernel(const unsigned char* __restrict__ keep, int n_users_block, int n_items, float* scores) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_users_block * n_items) return;
  if (!keep[g % n_items]) scores[g] = -INFINITY;
}

__device__ __forceinline__ unsigned orderable(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// per row the `cutoff` best items, best first (BaseRecommender.py:189-196); ties -> ascending item index.
// One CTA per row: MSB radix select of the cutoff-th key over 64-bit keys (score bits, ~index), then the survivors
// are ranked by counting (cutoff is small: <= 1024).
constexpr int TOPN_THREADS = 256;
constexpr int TOPN_MAX = 1024;
__global__ void __launch_bounds__(TOPN_THREADS) topn_rows_kernel(const float* __restrict__ scores, int n_rows, int n_items,
                                                                int cutoff, int* out_items, float* out_scores) {
  __shared__ int hist[2048];
  __shared__ int s_digit, s_need, s_cnt;
  __shared__ u64 cand[TOPN_MAX];
  const int tid = threadIdx.x;
  for (int row = blockIdx.x; row < n_rows; row += gridDim.x) {
    const float* L = scores + (size_t)row * n_items;
    const int keep = min(cutoff, n_items);
    u64 prefix = 0, mask = 0;
    int need = keep;
    if (keep < n_items) {
      for (int shift = 53;; shift -= 11) {
        const int sh = max(shift, 0), nb = shift >= 0 ? 11 : 11 + shift;
        for (int i = tid; i < 2048; i += TOPN_THREADS) hist[i] = 0;
        __syncthreads();
        for (int q = tid; q < n_items; q += TOPN_THREADS) {
          const u64 key = (((u64)orderable(L[q])) << 32) | (u64)(0xFFFFFFFFu - (unsigned)q);
          if ((key & mask) == prefix) atomicAdd(&hist[(int)((key >> sh) & ((1u << nb) - 1))], 1);
        }
        __syncthreads();
        if (tid < 32) {
          int local = 0;
          for (int b = 0; b < 64; ++b) local += hist[tid * 64 + b];
          int incl = local;
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            const int t = __shfl_down_sync(0xffffffffu, incl, off);
            if (tid + off < 32) incl += t;
          }
          int cum = incl - local;
          for (int b = 63; b >= 0; --b) {
            const int c = hist[tid * 64 + b];
            if (cum < need && cum + c >= need) { s_digit = tid * 64 + b; s_need = need - cum; }
            cum += c;
          }
        }
        __syncthreads();
        prefix |= ((u64)s_digit) << sh;
        mask |= ((u64)((1u << nb) - 1)) << sh;
        need = s_need;
        __syncthreads();
        if (shift <= 0) break;
      }
    }
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int q = tid; q < n_items; q += TOPN_THREADS) {
      const u64 key = (((u64)orderable(L[q])) << 32) | (u64)(0xFFFFFFFFu - (unsigned)q);
      if (key >= prefix) cand[atomicAdd(&s_cnt, 1)] = key;
    }
    __syncthreads();
    const int n = s_cnt;  // == keep
    for (int t = tid; t < n; t += TOPN_THREADS) {
      const u64 k = cand[t];
      int rank = 0;
      for (int q = 0; q < n; ++q) rank += cand[q] > k;
      const int item = (int)(0xFFFFFFFFu - (unsigned)k);
      out_items[(size_t)row * cutoff + rank] = item;
      out_scores[(size_t)row * cutoff + rank] = L[item];
    }
    for (int t = n + tid; t < cutoff; t += TOPN_THREADS) { out_items[(size_t)row * cutoff + t] = -1; out_scores[(size_t)row * cutoff + t] = -INFINITY; }
    __syncthreads();
  }
}

}  // namespace score
}  // namespace b200

using namespace b200;
using namespace b200::score;

extern "C" {

int b200_score_spmm_device(const int32_t* d_users, int n_users_block, const int32_t* d_a_ptr, const int32_t* d_a_idx,
                           const float* d_a_val, const int32_t* d_b_ptr, const int32_t* d_b_idx, const float* d_b_val,
                           int n_out_cols, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_a_ptr && d_b_val && d_out, "b200_score_spmm: NULL argument");
    B200_REQUIRE(n_users_block >= 0 && n_out_cols > 0, "b200_score_spmm: bad shape");
    if (n_users_block == 0) return;
    spmm_rows_kernel<<<std::min(n_users_block, sm_count() * 4), 512, 0, (cudaStream_t)stream>>>(
        d_users, n_users_block, d_a_ptr, d_a_idx, d_a_val, d_b_ptr, d_b_idx, d_b_val, n_out_cols, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_transpose_device(const float* d_in, int rows, int cols, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_in && d_out && rows > 0 && cols > 0, "b200_transpose: bad argument");
    transpose_kernel<<<dim3(div_up(cols, 32), div_up(rows, 32)), dim3(32, 8), 0, (cudaStream_t)stream>>>(d_in, rows, cols, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_score_mf_device(const int32_t* d_users, int n_users_block, const float* d_user_factors, const float* d_item_factors_T,
                         int n_factors, int n_items, const float* d_user_bias, const float* d_item_bias,
                         const float* d_global_bias, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_user_factors && d_item_factors_T && d_out, "b200_score_mf: NULL argument");
    B200_REQUIRE(n_factors >= 1 && n_items > 0 && n_users_block >= 0, "b200_score_mf: bad shape");
    B200_REQUIRE((d_global_bias == nullptr) == (d_user_bias == nullptr) && (d_user_bias == nullptr) == (d_item_bias == nullptr),
                 "b200_score_mf: biases must be all given or all NULL");
    if (n_users_block == 0) return;
    const size_t smem = (size_t)UT * n_factors * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "b200_score_mf: n_factors=%d too large", n_factors);
    mf_scores_kernel<<<dim3(div_up(n_items, 256), div_up(n_users_block, UT)), 256, smem, (cudaStream_t)stream>>>(
        d_users, n_users_block, d_user_factors, d_item_factors_T, n_factors, n_items, d_user_bias, d_item_bias, d_global_bias, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_score_mask_device(const int32_t* d_users, int n_users_block, const int32_t* d_urm_ptr, const int32_t* d_urm_idx,
                           const unsigned char* d_items_keep, int n_items, float* d_scores, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_scores && n_items > 0 && n_users_block >= 0, "b200_score_mask: bad argument");
    if (n_users_block == 0) return;
    cudaStream_t st = (cudaStream_t)stream;
    if (d_items_keep) {
      mask_items_kernel<<<div_up((long long)n_users_block * n_items, 256), 256, 0, st>>>(d_items_keep, n_users_block, n_items, d_scores);
      count_launch();
    }
    if (d_users && d_urm_ptr && d_urm_idx) {
      mask_seen_kernel<<<div_up((long long)n_users_block * 32, 256), 256, 0, st>>>(d_users, n_users_block, d_urm_ptr, d_urm_idx, n_items, d_scores);
      count_launch();
    }
    B200_CUDA(cudaGetLastError());
  });
}

int b200_score_topn_device(const float* d_scores, int n_rows, int n_items, int cutoff, int32_t* d_items, float* d_item_scores,
                           void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_scores && d_items && d_item_scores, "b200_score_topn: NULL argument");
    B200_REQUIRE(cutoff >= 1 && cutoff <= TOPN_MAX, "b200_score_topn: cutoff must be in [1, %d]", TOPN_MAX);
    if (n_rows == 0) return;
    topn_rows_kernel<<<std::min(n_rows, sm_count() * 8), TOPN_THREADS, 0, (cudaStream_t)stream>>>(d_scores, n_rows, n_items, cutoff,
                                                                                                  d_items, d_item_scores);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

}  // extern "C"
