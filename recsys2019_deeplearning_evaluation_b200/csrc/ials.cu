// K4: implicit-ALS half epochs (per-row normal equations), sm_90a.
//
// Replaces MatrixFactorization/IALSRecommender.py:137-201: for every warm user (then every warm item)
//     A = Y_p^T diag(c - 1) Y_p,   B = Y^T Y + A + reg * I,   x = B^{-1} Y_p^T c
// with Y the other side's factors, p the row's interaction profile and c its confidences (:170-201).
//
// One CTA per row.  The f x f matrix A is accumulated in REGISTERS: the 256 threads form a 16 x 16 grid, thread
// (ty, tx) owns the lower-triangular entries (r, c) with r = ty + 16 i, c = tx + 16 j, j <= i, and consumes the
// profile's factor rows from a shared-memory tile that all threads fill with coalesced loads.  B is then completed in
// shared memory in packed lower-triangular form, factorised by an in-place Cholesky and used for the two triangular
// solves (the reference forms the explicit inverse, :201; the solution is the same).  Y^T Y is accumulated by the
// same register tiling over row chunks with fp64 atomics.
// Everything is fp64 like the reference (:204-210): with the reference's all-positive initial factors the systems
// have condition numbers ~1e6, beyond what an fp32 factorisation resolves to the 1e-4 parity bar.
// CUDA-core fp64; the tensor-core kernel for n_factors >= 128 is ials_v2.cuh (DESIGN.md K4).
// n_factors <= 208: the packed fp64 matrix lives in shared memory.  208 < n_factors <= 256 (BASELINE.json configs[3]):
// the first R rows of the packed matrix stay in shared memory, the last ones in a per-CTA slab of global memory, and
// the register-tiled Gram accumulation takes two passes over the profile (136 fp64 accumulators do not fit one).
#include <algorithm>
#include <stdlib.h>

#include "common.cuh"

namespace b200 {
namespace ials {

constexpr int THREADS = 256;
constexpr int TROWS = 8;  // factor rows of the profile staged per tile

__device__ __forceinline__ int pidx(int r, int c) { return r * (r + 1) / 2 + c; }  // packed lower, c <= r

// Packed lower-triangular fp64 matrix of one CTA: rows below R live in shared memory, rows R.. in a per-CTA slab of
// global memory (L1/L2 resident).  HYB = false: everything is in shared memory (n_factors <= 208).
template <bool HYB>
struct Packed {
  double* s;
  double* g;   // row r >= R starts at g[pidx(r, 0) - pidx(R, 0)]
  int R, baseR;
  __device__ __forceinline__ double& operator()(int r, int c) const {
    if (HYB && r >= R) return g[pidx(r, c) - baseR];
    return s[pidx(r, c)];
  }
};

// acc[i - I0][j] (I0 <= i < I1, j <= i) += w * y[r_i] * y[c_j] for the rows in the tile
template <int FB, int I0, int I1>
__device__ __forceinline__ void rank_update(double (&acc)[I1 - I0][FB], const double* tile, const double* wt, int nrows, int f,
                                            int ty, int tx) {
  for (int t = 0; t < nrows; ++t) {
    const double* y = tile + t * f;
    const double w = wt[t];
    double yr[I1 - I0], yc[I1];
#pragma unroll
    for (int i = I0; i < I1; ++i) {
      const int r = ty + 16 * i;
      yr[i - I0] = r < f ? y[r] * w : 0.0;
    }
#pragma unroll
    for (int j = 0; j < I1; ++j) {
      const int c = tx + 16 * j;
      yc[j] = c < f ? y[c] : 0.0;
    }
#pragma unroll
    for (int i = I0; i < I1; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) acc[i - I0][j] += yr[i - I0] * yc[j];
  }
}

// YtY[r, c] (full symmetric f x f, fp64) += sum over rows n in this CTA's chunk of Y[n, r] * Y[n, c], for the row
// blocks I0 <= i < I1 of the 16 x 16 thread tiling (one launch for FB <= 13, two for FB = 16: register budget)
template <int FB, int I0, int I1>
__global__ void __launch_bounds__(THREADS) gram_kernel(const double* __restrict__ Y, int n_rows, int f, double* YtY) {
  extern __shared__ double sm[];
  double* tile = sm;               // TROWS x f
  double* wt = sm + TROWS * f;     // TROWS
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  double acc[I1 - I0][FB];
#pragma unroll
  for (int i = 0; i < I1 - I0; ++i)
#pragma unroll
    for (int j = 0; j < FB; ++j) acc[i][j] = 0.0;
  const int per = (n_rows + gridDim.x - 1) / gridDim.x;
  const int lo = blockIdx.x * per, hi = min(n_rows, lo + per);
  for (int n0 = lo; n0 < hi; n0 += TROWS) {
    const int nr = min(TROWS, hi - n0);
    __syncthreads();
    for (int e = tid; e < nr * f; e += THREADS) tile[e] = Y[(size_t)n0 * f + e];
    if (tid < nr) wt[tid] = 1.0;
    __syncthreads();
    rank_update<FB, I0, I1>(acc, tile, wt, nr, f, ty, tx);
  }
#pragma unroll
  for (int i = I0; i < I1; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      const int r = ty + 16 * i, c = tx + 16 * j;
      const double v = acc[i - I0][j];
      if (r < f && c < f && c <= r && v != 0.0) {
        atomicAdd(YtY + (size_t)r * f + c, v);
        if (c != r) atomicAdd(YtY + (size_t)c * f + r, v);
      }
    }
}

// One pass over the profile of `row`: B(r, c) = A(r, c) + YtY(r, c) + reg [r == c] for the row blocks I0 <= i < I1, and
// (RHS) rhs = Y_p^T c.
template <int FB, int I0, int I1, bool HYB, bool RHS>
__device__ __forceinline__ void profile_pass(const Packed<HYB>& B, double* tile, double* wt, double* cw, double* rhs, int p0, int p1,
                                             const int* __restrict__ idx, const float* __restrict__ conf,
                                             const double* __restrict__ Y, const double* __restrict__ YtY, int f, double reg) {
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  double acc[I1 - I0][FB];
#pragma unroll
  for (int i = 0; i < I1 - I0; ++i)
#pragma unroll
    for (int j = 0; j < FB; ++j) acc[i][j] = 0.0;
  double my_rhs = 0.0;  // thread tid < f owns rhs[tid]
  for (int k0 = p0; k0 < p1; k0 += TROWS) {
    const int nr = min(TROWS, p1 - k0);
    __syncthreads();
    for (int e = tid; e < nr * f; e += THREADS) {
      const int t = e / f, q = e % f;
      tile[e] = Y[(size_t)idx[k0 + t] * f + q];
    }
    if (tid < nr) { const double c = (double)conf[k0 + tid]; wt[tid] = c - 1.0; cw[tid] = c; }
    __syncthreads();
    rank_update<FB, I0, I1>(acc, tile, wt, nr, f, ty, tx);
    if (RHS && tid < f)
      for (int t = 0; t < nr; ++t) my_rhs += cw[t] * tile[t * f + tid];  // Y_p^T c (:201)
  }
  __syncthreads();
  // B = YtY + A + reg I (:199), packed lower
#pragma unroll
  for (int i = I0; i < I1; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      const int r = ty + 16 * i, c = tx + 16 * j;
      if (r < f && c <= r) B(r, c) = acc[i - I0][j] + YtY[(size_t)r * f + c] + (r == c ? reg : 0.0);
    }
  if (RHS && tid < f) rhs[tid] = my_rhs;
}

template <int FB, int SPLIT, bool HYB>
__global__ void __launch_bounds__(THREADS) ials_rows_kernel(const int* __restrict__ rows, int n_solve, const int* __restrict__ ptr,
                                                            const int* __restrict__ idx, const float* __restrict__ conf,
                                                            const double* __restrict__ Y, const double* __restrict__ YtY, int f,
                                                            double reg, double* X, int* info, int R, double* gslab, int gstride) {
  extern __shared__ double sm[];
  const int nps = R * (R + 1) / 2;       // packed entries kept in shared memory
  double* tile = sm + nps;               // TROWS x f
  double* wt = tile + TROWS * f;         // TROWS: c - 1
  double* rhs = wt + TROWS;              // f
  double* cw = rhs + f;                  // TROWS: c
  Packed<HYB> B;
  B.s = sm; B.g = HYB ? gslab + (size_t)blockIdx.x * gstride : nullptr; B.R = R; B.baseR = nps;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  for (int s = blockIdx.x; s < n_solve; s += gridDim.x) {
    const int row = rows[s];
    const int p0 = ptr[row], p1 = ptr[row + 1];
    profile_pass<FB, 0, SPLIT, HYB, true>(B, tile, wt, cw, rhs, p0, p1, idx, conf, Y, YtY, f, reg);
    if constexpr (SPLIT < FB)  // second pass over the profile for the remaining row blocks (register budget at f > 208)
      profile_pass<FB, SPLIT, FB, HYB, false>(B, tile, wt, cw, rhs, p0, p1, idx, conf, Y, YtY, f, reg);
    __syncthreads();
    // in-place Cholesky (right-looking)
    for (int j = 0; j < f; ++j) {
      if (tid == 0) {
        const double d = B(j, j);
        if (!(d > 0.0)) atomicExch(info, row + 1);
        B(j, j) = sqrt(fmax(d, 1e-300));
      }
      __syncthreads();
      const double djj = B(j, j);
      for (int r = j + 1 + tid; r < f; r += THREADS) B(r, j) /= djj;
      __syncthreads();
      // rows r > j, columns j < c <= r: thread-strided over rows and columns (16 x 16 grid)
      for (int r = j + 1 + ty; r < f; r += 16) {
        const double lrj = B(r, j);
        for (int c = j + 1 + tx; c <= r; c += 16) B(r, c) -= lrj * B(c, j);
      }
      __syncthreads();
    }
    // forward solve L z = rhs, then backward L^T x = z (one warp; f is small)
    if (tid < 32) {
      for (int r = 0; r < f; ++r) {
        double part = 0.0;
        for (int c = tid; c < r; c += 32) part += B(r, c) * rhs[c];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        if (tid == 0) rhs[r] = (rhs[r] - part) / B(r, r);
        __syncwarp();
      }
      for (int r = f - 1; r >= 0; --r) {
        double part = 0.0;
        for (int c = r + 1 + tid; c < f; c += 32) part += B(c, r) * rhs[c];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        if (tid == 0) rhs[r] = (rhs[r] - part) / B(r, r);
        __syncwarp();
      }
    }
    __syncthreads();
    if (tid < f) X[(size_t)row * f + tid] = rhs[tid];
    __syncthreads();
  }
}

template <int FB, int SPLIT>
void run(cudaStream_t st, const int* rows, int n_solve, const int* ptr, const int* idx, const float* conf, const double* Y,
         int n_other, int f, double reg, double* X, double* YtY, int* info) {
  const size_t smem_g = sizeof(double) * ((size_t)TROWS * f + TROWS);
  B200_CUDA(cudaMemsetAsync(YtY, 0, sizeof(double) * (size_t)f * f, st));
  const int grid_g = std::max(1, std::min(sm_count() * 4, (n_other + 63) / 64));
  gram_kernel<FB, 0, SPLIT><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY);
  count_launch();
  if constexpr (SPLIT < FB) {
    gram_kernel<FB, SPLIT, FB><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY);
    count_launch();
  }
  // rows of the packed matrix that fit the shared memory next to the tile; the rest go to a global slab per CTA
  constexpr bool HYB = SPLIT < FB;
  int dev = 0, max_smem = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t other = sizeof(double) * ((size_t)TROWS * f + 2 * TROWS + f);
  int R = f;
  while (R > 0 && sizeof(double) * ((size_t)R * (R + 1) / 2) + other > (size_t)max_smem) --R;
  B200_REQUIRE(HYB || R == f, "b200_ials_half_epoch: %d factors do not fit %d bytes of shared memory", f, max_smem);
  const size_t smem = sizeof(double) * ((size_t)R * (R + 1) / 2) + other;
  auto kern = ials_rows_kernel<FB, SPLIT, HYB>;
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, THREADS, smem));
  const int grid = std::max(1, std::min(n_solve, sm_count() * std::max(per_sm, 1)));
  const int gstride = f * (f + 1) / 2 - R * (R + 1) / 2;
  DevBuf<double> gslab;
  if (gstride > 0) gslab.alloc((size_t)grid * gstride);
  kern<<<grid, THREADS, smem, st>>>(rows, n_solve, ptr, idx, conf, Y, YtY, f, reg, X, info, R, gslab.get(), gstride);
  B200_CUDA(cudaGetLastError());
  count_launch();
  if (gstride > 0) B200_CUDA(cudaStreamSynchronize(st));  // the slab is freed on return
}

}  // namespace ials
}  // namespace b200

#include "ials_v2.cuh"

namespace b200 {
namespace ials {

// Tensor-core half epoch, second generation (ials_v2.cuh, n_factors <= 256); false when a row asked for the fp64 path.
bool run_v2(cudaStream_t st, const int* rows, int n_solve, const int* ptr, const int* idx, const float* conf, const double* Y,
            int n_other, int f, double reg, double* X, double* YtY, int* info) {
  const size_t smem_g = sizeof(double) * ((size_t)TROWS * f + TROWS);
  B200_CUDA(cudaMemsetAsync(YtY, 0, sizeof(double) * (size_t)f * f, st));
  const int grid_g = std::max(1, std::min(sm_count() * 4, (n_other + 63) / 64));
  if (f <= 32) { gram_kernel<2, 0, 2><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch(); }
  else if (f <= 64) { gram_kernel<4, 0, 4><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch(); }
  else if (f <= 128) { gram_kernel<8, 0, 8><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch(); }
  else if (f <= 208) { gram_kernel<13, 0, 13><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch(); }
  else {
    gram_kernel<16, 0, 11><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch();
    gram_kernel<16, 11, 16><<<grid_g, THREADS, smem_g, st>>>(Y, n_other, f, YtY); count_launch();
  }
  DevBuf<int> redo(1);
  B200_CUDA(cudaMemsetAsync(redo.get(), 0, sizeof(int), st));
  const size_t smem = ials2::smem_bytes(f);
  auto kern = f > 128 ? ials2::ials_rows_v2_kernel<true> : ials2::ials_rows_v2_kernel<false>;
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = std::max(1, std::min(n_solve, sm_count()));
  kern<<<grid, ials2::T, smem, st>>>(rows, n_solve, ptr, idx, conf, Y, YtY, f, reg, X, info, redo.get(), 2);
  B200_CUDA(cudaGetLastError());
  count_launch();
  int h_redo = 0;
  B200_CUDA(cudaMemcpyAsync(&h_redo, redo.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  return h_redo == 0;
}

}  // namespace ials
}  // namespace b200

using namespace b200;

extern "C" {

int b200_ials_half_epoch_device(const int32_t* d_rows, int n_solve, const int32_t* d_ptr, const int32_t* d_idx, const float* d_conf,
                                const double* d_Y, int n_other, int n_factors, double reg, double* d_X, double* d_YtY_work,
                                void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_rows && d_ptr && d_idx && d_conf && d_Y && d_X && d_YtY_work, "b200_ials_half_epoch: NULL argument");
    B200_REQUIRE(n_factors >= 1 && n_factors <= 256, "b200_ials_half_epoch: n_factors must be in [1, 256] (got %d)", n_factors);
    B200_REQUIRE(n_solve >= 0 && n_other > 0, "b200_ials_half_epoch: bad shape");
    if (n_solve == 0) return;
    cudaStream_t st = (cudaStream_t)stream;
    DevBuf<int> info(1);
    B200_CUDA(cudaMemsetAsync(info.get(), 0, sizeof(int), st));
    const int f = n_factors;
    // tensor-core path, second generation (ials_v2.cuh): the default whenever the other side has at least 4 x n_factors rows
    // (well-conditioned systems; B200REC_IALS_V2=0 switches it off); a row whose refinement does not contract sends the half
    // epoch back to the fp64 kernel below
    const int v2_env = getenv("B200REC_IALS_V2") ? atoi(getenv("B200REC_IALS_V2")) : -1;  // 0 off, 1 every size, unset: where it wins
    const bool want_v2 = v2_env == 1 || (v2_env != 0 && f >= 128);
    if (want_v2 && n_other >= 4 * f) {
      if (ials::run_v2(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get())) {
        int h_info = 0;
        B200_CUDA(cudaMemcpyAsync(&h_info, info.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        B200_REQUIRE(h_info == 0, "b200_ials_half_epoch: normal equations of row %d are not positive definite", h_info - 1);
        return;
      }
      B200_CUDA(cudaMemsetAsync(info.get(), 0, sizeof(int), st));  // redo the half epoch in fp64
    }
    if (f <= 32) ials::run<2, 2>(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get());
    else if (f <= 64) ials::run<4, 4>(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get());
    else if (f <= 128) ials::run<8, 8>(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get());
    else if (f <= 208) ials::run<13, 13>(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get());
    else ials::run<16, 11>(st, d_rows, n_solve, d_ptr, d_idx, d_conf, d_Y, n_other, f, reg, d_X, d_YtY_work, info.get());
    int h_info = 0;
    B200_CUDA(cudaMemcpyAsync(&h_info, info.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_REQUIRE(h_info == 0, "b200_ials_half_epoch: normal equations of row %d are not positive definite", h_info - 1);
  });
}

}  // extern "C"
