// K1b: top-K along the rows or columns of a dense fp32 matrix resident in HBM, sm_90a.
//
// Replaces the two numpy top-K loops the reference runs over item-item matrices:
//   * Base/Recommender_utils.py:55-122 similarityMatrixTopK -- per COLUMN, the k largest of the NON-ZERO values
//     (negatives survive when there are fewer than k positives)                       -> mode B200_TOPK_NONZERO
//   * SLIM_BPR_Cython_Epoch.pyx:340-388 get_S / Triangular_Matrix.get_scipy_csr :1335-1415 -- per ROW, the k
//     largest over ALL cells, zeros then dropped (zeros outrank negatives)            -> mode B200_TOPK_ZEROS_OUTRANK
//   * SLIM_ElasticNet/SLIMElasticNetRecommender.py:99-107 -- per item, the min(nnz - 1, k) largest of the non-zero
//     coefficients: a line with <= k non-zeros loses its smallest one                  -> mode 2
// One CTA per line; the line is streamed from HBM/L2 once per radix pass (select.cuh, 11-bit digits over the 64-bit key
// value-bits << 32 | ~index, so ties resolve to the ascending index); survivors are written as a [lines, K] table.
// NaN is a non-zero cell and ranks where the reference's numpy call puts it: above +inf in mode 0 (argsort ascending,
// last k), below -inf in modes 1 and 2 (argpartition of the negated line). A line never emits more than K entries:
// cells whose key equals the threshold (a duplicated (index, value) entry of a compressed line) are taken only as many
// times as the selection still needs.
#include <algorithm>

#include "common.cuh"
#include "select.cuh"

namespace b200 {
namespace dtk {

typedef unsigned long long u64;
constexpr int THREADS = 256;
constexpr int BINS = 2048;

// SPARSE: line l is the segment [ptr[l], ptr[l+1]) of (sidx, M); its cells are the stored entries and the implicit
// zeros of a length-n_inner line.  Residency: 8 CTAs per SM for compressed lines (32 registers: the grid of sm_count * 8
// is resident at once), 6 for dense ones (40 registers).
template <bool SPARSE>
__global__ void __launch_bounds__(THREADS, SPARSE ? 8 : 6)
    topk_lines_kernel(const float* __restrict__ M, const int* __restrict__ ptr, const int* __restrict__ sidx, int n_lines,
                      int n_inner_dense, long long stride_line, long long stride_inner, int K, int mode, int* out_idx,
                      float* out_val, int* out_cnt, int idx_off = 0) {
  __shared__ CtaSelectSmem<BINS> sel;
  __shared__ int s_cnt, s_tie, s_npos, s_nneg, s_nnan;
  const int tid = threadIdx.x, lane = tid & 31;
  const bool nan_high = mode == 0;
  for (int line = blockIdx.x; line < n_lines; line += gridDim.x) {
    const float* L = SPARSE ? M + ptr[line] : M + (long long)line * stride_line;
    const int* LI = SPARSE ? sidx + ptr[line] : nullptr;
    const int n_inner = SPARSE ? ptr[line + 1] - ptr[line] : n_inner_dense;
    if (SPARSE) stride_inner = 1;
    if (tid == 0) { s_npos = 0; s_nneg = 0; s_nnan = 0; s_cnt = 0; s_tie = 0; }
    __syncthreads();
    int npos = 0, nneg = 0, nnan = 0;
    for (int q = tid; q < n_inner; q += THREADS) {
      const float v = L[(long long)q * stride_inner];
      npos += v > 0.f;
      nneg += v < 0.f;
      nnan += v != v;
    }
    npos = __reduce_add_sync(0xffffffffu, npos);
    nneg = __reduce_add_sync(0xffffffffu, nneg);
    nnan = __reduce_add_sync(0xffffffffu, nnan);
    if (lane == 0) { atomicAdd(&s_npos, npos); atomicAdd(&s_nneg, nneg); atomicAdd(&s_nnan, nnan); }
    __syncthreads();
    npos = s_npos; nneg = s_nneg; nnan = s_nnan;
    const int nnz = npos + nneg + nnan;  // the cells with v != 0
    const int nzero = n_inner_dense - nnz;
    int keep;  // how many non-zero cells survive
    if (mode == 0) keep = min(K, nnz);                                           // similarityMatrixTopK
    else if (mode == 2) keep = drop_last_keep(K, nnz);                           // SLIMElasticNetRecommender.py:103
    else keep = min(K, npos) + min(nneg + nnan, max(0, K - npos - nzero));        // zeros outrank negatives, NaN last
    keep = min(keep, K);  // nzero < 0 when a compressed line holds more entries than n
    u64 thr = 0;
    int ties = keep;  // how many cells with key == thr are taken
    if (keep > 0 && keep < nnz) {
      const auto sel_key = [&](int q, u64& key) {
        const float v = L[(long long)q * stride_inner];
        if (v != 0.f) key = line_key(v, SPARSE ? LI[q] : q + idx_off, nan_high);
        return v != 0.f;
      };
      const Threshold<u64> t = radix_select<u64, 11, false>(CtaSelect<THREADS, BINS>(sel), n_inner, keep, sel_key);
      thr = t.thr;
      ties = t.need;  // 1 unless entries repeat (index, value): keys are distinct within a line otherwise
    }
    // emit: the keys above thr, then at most `ties` of the keys equal to it
    if (keep > 0) {
      for (int q = tid; q < n_inner; q += THREADS) {
        const float v = L[(long long)q * stride_inner];
        if (v != 0.f) {
          const int qi = SPARSE ? LI[q] : q + idx_off;
          const u64 key = line_key(v, qi, nan_high);
          if (key > thr || (key == thr && atomicAdd(&s_tie, 1) < ties)) {
            const int pos = atomicAdd(&s_cnt, 1);
            out_idx[(size_t)line * K + pos] = qi;
            out_val[(size_t)line * K + pos] = v;
          }
        }
      }
    }
    __syncthreads();
    const int cnt = s_cnt;
    for (int t = cnt + tid; t < K; t += THREADS) { out_idx[(size_t)line * K + t] = -1; out_val[(size_t)line * K + t] = 0.f; }
    if (tid == 0) out_cnt[line] = cnt;
    __syncthreads();
  }
}

}  // namespace dtk
}  // namespace b200

using namespace b200;

extern "C" {

int b200_dense_topk_device(const float* d_matrix, int n, int K, int along_columns, int mode, int32_t* d_idx, float* d_val,
                           int32_t* d_cnt, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_matrix && d_idx && d_val && d_cnt, "b200_dense_topk: NULL argument");
    B200_REQUIRE(n > 0 && K > 0 && K <= n, "b200_dense_topk: need 0 < K <= n (got K=%d n=%d)", K, n);
    B200_REQUIRE(mode >= 0 && mode <= 2, "b200_dense_topk: unknown mode %d", mode);
    cudaStream_t st = (cudaStream_t)stream;
    const long long sl = along_columns ? 1 : n, si = along_columns ? n : 1;
    dtk::topk_lines_kernel<false><<<std::min(n, sm_count() * 8), dtk::THREADS, 0, st>>>(d_matrix, nullptr, nullptr, n, n, sl, si, K, mode, d_idx, d_val, d_cnt);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_dense_topk_rect_device(const float* d_matrix, int n_lines, int n_inner, int64_t stride_line, int64_t stride_inner, int index_offset,
                                int K, int mode, int32_t* d_idx, float* d_val, int32_t* d_cnt, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_matrix && d_idx && d_val && d_cnt, "b200_dense_topk_rect: NULL argument");
    B200_REQUIRE(n_lines > 0 && n_inner > 0 && K > 0, "b200_dense_topk_rect: bad shape");
    // mode 1 counts a line's zeros among its n_inner cells, so it is only right for whole lines (a slab of full rows), never
    // for a column slab of a sharded matrix, whose other shards' zeros are not visible here
    B200_REQUIRE(mode == 0 || mode == 1, "b200_dense_topk_rect: mode must be 0 or 1 (got %d)", mode);
    dtk::topk_lines_kernel<false><<<std::min(n_lines, sm_count() * 8), dtk::THREADS, 0, (cudaStream_t)stream>>>(
        d_matrix, nullptr, nullptr, n_lines, n_inner, (long long)stride_line, (long long)stride_inner, K, mode, d_idx, d_val, d_cnt, index_offset);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_sparse_topk_device(int n, const int32_t* d_ptr, const int32_t* d_line_idx, const float* d_vals, int K, int mode,
                            int32_t* d_idx, float* d_val, int32_t* d_cnt, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_ptr && d_idx && d_val && d_cnt, "b200_sparse_topk: NULL argument");
    B200_REQUIRE(n > 0 && K > 0 && K <= n, "b200_sparse_topk: need 0 < K <= n (got K=%d n=%d)", K, n);
    B200_REQUIRE(mode == 0 || mode == 1, "b200_sparse_topk: unknown mode %d", mode);
    cudaStream_t st = (cudaStream_t)stream;
    dtk::topk_lines_kernel<true><<<std::min(n, sm_count() * 8), dtk::THREADS, 0, st>>>(d_vals, d_ptr, d_line_idx, n, n, 0, 1, K, mode,
                                                                                       d_idx, d_val, d_cnt);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

}  // extern "C"
