// URM feature weighting in front of the KNN similarity (SURVEY.md 8(f).3), sm_90a.
//
// Replaces Base/IR_feature_weighting.py:13-78 as KNN/ItemKNNCFRecommender.py:42-50 and KNN/UserKNNCFRecommender.py:43-51
// apply it: okapi_BM_25(URM.T).T and TF_IDF(URM.T).T -- items are the "documents" (rows of URM.T), users the "terms".
// In URM orientation (CSR, row = user u, column = item i, value r):
//     idf[u]         = log(n_items / (1 + len_u))                                     (IR_feature_weighting.py:37,71)
//     TF-IDF         : r' = sqrt(r) * idf[u]                                           (:74)
//     BM25           : len_norm[i] = (1 - B) + B * colsum_i / mean(colsum)             (:40-43)
//                      den = K1 * len_norm[i] + r,  den == 0 -> 1e-9                   (:46-47)
//                      r' = r * (K1 + 1) / den * idf[u]                                (:49)
// Element-wise and HBM-bound: one pass for the column sums (fp64 atomics), one warp-per-row pass that rewrites the values
// in place.  Arithmetic in fp64 (the reference mixes fp32 sums with fp64 idf and casts the result to fp32).
#include "common.cuh"

namespace b200 {
namespace weighting {

__global__ void colsum_kernel(const int* __restrict__ idx, const float* __restrict__ data, long long nnz, double* colsum) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(colsum + idx[i], (double)data[i]);
}

// total[0] = sum of colsum (one block)
__global__ void total_kernel(const double* __restrict__ colsum, int n_cols, double* total) {
  __shared__ double part[32];
  double s = 0.0;
  for (int j = threadIdx.x; j < n_cols; j += blockDim.x) s += colsum[j];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (threadIdx.x == 0) total[0] = s;
  }
}

// mode 0 = BM25, 1 = TF-IDF; one warp per row (user)
__global__ void apply_kernel(int mode, int n_rows, int n_cols, const int* __restrict__ ptr, const int* __restrict__ idx,
                             float* data, const double* __restrict__ colsum, const double* __restrict__ total, double K1,
                             double B) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_rows) return;
  const int s = ptr[warp], e = ptr[warp + 1];
  if (e <= s) return;
  const double idf = log((double)n_cols / (1.0 + (double)(e - s)));
  const double avg = mode == 0 ? total[0] / (double)n_cols : 1.0;
  for (int q = s + lane; q < e; q += 32) {
    const double r = (double)data[q];
    double v;
    if (mode == 0) {
      const double ln = (1.0 - B) + B * colsum[idx[q]] / avg;
      double den = K1 * ln + r;
      if (den == 0.0) den += 1e-9;
      v = r * (K1 + 1.0) / den * idf;
    } else {
      v = sqrt(r) * idf;
    }
    data[q] = (float)v;
  }
}

}  // namespace weighting
}  // namespace b200

using namespace b200;

extern "C" {

int b200_feature_weighting_device(int mode, int n_users, int n_items, int64_t nnz, const int32_t* d_indptr, const int32_t* d_indices,
                                  float* d_data, float K1, float B, void* stream) {
  return guarded([&] {
    B200_REQUIRE(mode == B200_WEIGHT_BM25 || mode == B200_WEIGHT_TFIDF, "b200_feature_weighting: unknown mode %d", mode);
    B200_REQUIRE(n_users > 0 && n_items > 0 && nnz >= 0, "b200_feature_weighting: bad shape");
    B200_REQUIRE(d_indptr && (nnz == 0 || (d_indices && d_data)), "b200_feature_weighting: NULL argument");
    if (mode == B200_WEIGHT_BM25) {  // IR_feature_weighting.py:22-23
      B200_REQUIRE(B > 0.f && B < 1.f, "okapi_BM_25: B must be in (0,1)");
      B200_REQUIRE(K1 > 0.f, "okapi_BM_25: K1 must be > 0");
    }
    if (nnz == 0) return;
    cudaStream_t st = (cudaStream_t)stream;
    DevBuf<double> colsum, total(1);
    if (mode == B200_WEIGHT_BM25) {
      colsum.alloc((size_t)n_items);
      B200_CUDA(cudaMemsetAsync(colsum.get(), 0, sizeof(double) * (size_t)n_items, st));
      weighting::colsum_kernel<<<sm_count() * 8, 256, 0, st>>>(d_indices, d_data, nnz, colsum.get());
      weighting::total_kernel<<<1, 1024, 0, st>>>(colsum.get(), n_items, total.get());
      count_launch(2);
    }
    weighting::apply_kernel<<<div_up((long long)n_users * 32, 256), 256, 0, st>>>(mode, n_users, n_items, d_indptr, d_indices, d_data,
                                                                                  colsum.get(), total.get(), (double)K1, (double)B);
    B200_CUDA(cudaGetLastError());
    count_launch();
    B200_CUDA(cudaStreamSynchronize(st));  // the scratch buffers are freed on return
  });
}

}  // extern "C"
