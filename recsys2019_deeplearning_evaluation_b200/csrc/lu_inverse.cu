// Inverse of a general (non-singular) matrix in fp64 through a blocked LU factorisation with partial pivoting, sm_90a.
//
// The EASE_R inverse (ease.cu) of a Gram matrix that is not positive definite: the reference's np.linalg.inv factors any
// non-singular matrix by LU (LAPACK dgetrf / dgetri, in float64 even for a float32 input), and EASE_R's popularity-based
// diagonal (EASE_R_Recommender.py:62-63) leaves explicit-rating Grams indefinite at common l2_norm values.  These systems
// reach cond ~1e7, so the factorisation is fp64 throughout; every O(n^3) step is a GEMM on the FP64 tensor cores
// (dgemm_tc.cuh).  NB = 128 (the GEMM tile).
//   1. getrf, right-looking, one block column at a time:
//      a. the tall panel [k0:, k0:k0+NB] is factored with partial pivoting by one cooperative kernel that keeps every
//         CTA's share of the panel rows in global memory (L2-resident) and takes one grid barrier per column: the pivot
//         row (largest |a|, lowest row on ties: LAPACK's idamax rule) and the current diagonal row travel through small
//         double-buffered slots, so no CTA reads a row another CTA is rewriting;
//      b. the panel's row interchanges are applied to the columns left and right of it (laswp);
//      c. U12 = inv(L11) A12 as a GEMM (in place: each CTA reads only the tile it writes), A22 -= L21 U12.
//   2. getri: U^-1 and L^-1 (unit lower) by block diagonals, one batched GEMM pair per diagonal and factor, from the
//      128 x 128 diagonal-block inverses (one CTA each); then A^-1 = U^-1 L^-1 P as one GEMM with the K range of every
//      tile clipped to k >= max(row block, column block), its columns scattered by the row permutation P on the store.
// About 2 n^3 flops: 2n^3/3 for getrf, n^3/3 for each triangular inverse, 2n^3/3 for the product.
#include <algorithm>
#include <climits>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"
#include "dgemm_tc.cuh"

namespace cg = cooperative_groups;

namespace b200 {
namespace lu {

constexpr int NB = 128;       // panel width == GEMM tile
constexpr int PT = 256;       // threads per CTA of the panel kernel; also the largest panel grid
constexpr int TRI_SMEM = NB * (NB + 1) * 8;

__device__ __forceinline__ bool better(double v, int i, double bv, int bi) { return v > bv || (v == bv && i < bi); }

// (value, row) arg-max over the CTA, ties to the lower row; the result is valid in every thread after the call.
__device__ void block_argmax(double& v, int& i, double* sv, int* si) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double ov = __shfl_down_sync(0xffffffffu, v, off);
    const int oi = __shfl_down_sync(0xffffffffu, i, off);
    if (better(ov, oi, v, i)) { v = ov; i = oi; }
  }
  __syncthreads();  // sv / si may still be read by the previous call
  if (lane == 0) { sv[warp] = v; si[warp] = i; }
  __syncthreads();
  v = sv[0]; i = si[0];
  for (int w = 1; w < PT / 32; ++w)
    if (better(sv[w], si[w], v, i)) { v = sv[w]; i = si[w]; }
}

// Factors the panel P [rows, NB] (row-major, lda; the rows from the diagonal block down) with partial pivoting in place.
// Row i belongs to CTA i / ceil(rows / G).  ipiv[j] receives k0 + the pivot row of column j; info (if still 0) the
// 1-based global column of the first exactly zero pivot.  Scratch: cand_rows [2][G][NB], cand_val / cand_idx [2][G],
// diag_rows [2][NB] (slot j & 1 holds what step j reads).
__global__ void __launch_bounds__(PT) panel_getrf_kernel(double* P, int lda, int rows, int k0, int* ipiv, int* info, double* cand_rows,
                                                         double* cand_val, int* cand_idx, double* diag_rows) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double urow[NB], jrow[NB], lcol[PT], red_v[PT / 32];
  __shared__ int red_i[PT / 32];
  const int G = gridDim.x, c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rpc = (rows + G - 1) / G, r0 = min(rows, c * rpc), r1 = min(rows, r0 + rpc);

  // this CTA's candidate for the pivot of column col (rows >= col): |value|, row and the whole row; plus row col itself
  auto publish = [&](int col) {
    const int slot = col & 1;
    double v = -1.0;
    int i = INT_MAX;
    for (int r = max(r0, col) + tid; r < r1; r += PT) {
      const double a = fabs(P[(long long)r * lda + col]);
      if (better(a, r, v, i)) { v = a; i = r; }
    }
    block_argmax(v, i, red_v, red_i);
    if (tid == 0) { cand_val[slot * G + c] = v; cand_idx[slot * G + c] = i; }
    if (tid < NB) {
      if (v >= 0.0) cand_rows[((long long)slot * G + c) * NB + tid] = P[(long long)i * lda + tid];
      if (col >= r0 && col < r1) diag_rows[slot * NB + tid] = P[(long long)col * lda + tid];
    }
  };

  publish(0);
  grid.sync();
  for (int j = 0; j < NB; ++j) {
    const int slot = j & 1;
    double v = -1.0;
    int i = INT_MAX, w = -1;
    if (tid < G) { v = cand_val[slot * G + tid]; i = cand_idx[slot * G + tid]; }
    block_argmax(v, i, red_v, red_i);
    if (v >= 0.0) {  // the winning CTA: the lowest one whose candidate is the winning row (rows are owned by one CTA)
      w = i / rpc;
    } else {         // every candidate NaN: keep row j
      i = j;
    }
    const int p = i;
    const double* prow = w >= 0 ? cand_rows + ((long long)slot * G + w) * NB : diag_rows + slot * NB;
    if (tid < NB) { urow[tid] = prow[tid]; jrow[tid] = diag_rows[slot * NB + tid]; }
    __syncthreads();
    const double piv = urow[j];
    if (c == 0 && tid == 0) {
      ipiv[j] = k0 + p;
      if (piv == 0.0 && *info == 0) *info = k0 + j + 1;
    }
    // interchange rows j and p (the pivot row comes from its slot, row j from the diagonal slot)
    if (tid < NB) {
      if (j >= r0 && j < r1) P[(long long)j * lda + tid] = urow[tid];
      if (p != j && p >= r0 && p < r1) P[(long long)p * lda + tid] = jrow[tid];
    }
    __syncthreads();
    // multipliers of column j and the rank-1 update of columns j+1.. on this CTA's rows below the diagonal
    for (int base = max(r0, j + 1); base < r1; base += PT) {
      const int r = base + tid;
      if (r < r1) {
        double l = P[(long long)r * lda + j];
        if (piv != 0.0) l /= piv;  // a zero pivot leaves the (zero) column as it is, as LAPACK's dgetf2 does
        P[(long long)r * lda + j] = l;
        lcol[tid] = l;
      }
      __syncthreads();
      const int nrow = min(PT, r1 - base);
      for (int rr = warp; rr < nrow; rr += PT / 32) {
        double* row = P + (long long)(base + rr) * lda;
        const double l = lcol[rr];
        double x[NB / 32];  // all loads of the row before any store: one L2 round trip per row, not one per 32 columns
#pragma unroll
        for (int q = 0; q < NB / 32; ++q) {
          const int k = lane + 32 * q;
          x[q] = k > j ? row[k] : 0.0;
        }
#pragma unroll
        for (int q = 0; q < NB / 32; ++q) {
          const int k = lane + 32 * q;
          if (k > j) row[k] = fma(-l, urow[k], x[q]);
        }
      }
      __syncthreads();
    }
    if (j + 1 < NB) publish(j + 1);
    grid.sync();
  }
}

// Applies the row interchanges of panel k0 (ipiv[k0 .. k0+NB), in order) to every column outside the panel.
__global__ void laswp_kernel(double* A, int lda, int n_cols, int k0, const int* __restrict__ ipiv) {
  __shared__ int piv[NB];
  if (threadIdx.x < NB) piv[threadIdx.x] = ipiv[k0 + threadIdx.x];
  __syncthreads();
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= n_cols || (col >= k0 && col < k0 + NB)) return;
  for (int j = 0; j < NB; ++j) {
    const int p = piv[j];
    if (p != k0 + j) {
      double* a = A + (long long)(k0 + j) * lda + col;
      double* b = A + (long long)p * lda + col;
      const double t = *a;
      *a = *b;
      *b = t;
    }
  }
}

// Diagonal block blockIdx.x of the LU factors in A (lda): the inverse of its unit-lower part into Linv and of its upper
// part into Uinv (each a dense NB x NB block at the same block position, leading dimension ldo; either may be null).
// One column per thread: threads 0..127 forward substitution for L, 128..255 back substitution for U.
__global__ void __launch_bounds__(2 * NB) tri_inv_blocks_kernel(const double* __restrict__ A, int lda, double* Linv, double* Uinv,
                                                                int ldo) {
  extern __shared__ double T[];  // NB x (NB + 1)
  constexpr int LD = NB + 1;
  const long long blk = (long long)blockIdx.x * NB;
  for (int e = threadIdx.x; e < NB * NB; e += 2 * NB) {
    const int r = e / NB, cc = e % NB;
    T[r * LD + cc] = A[(blk + r) * lda + blk + cc];
  }
  __syncthreads();
  const int c = threadIdx.x & (NB - 1);
  if (threadIdx.x < NB) {
    if (!Linv) return;
    double* X = Linv + blk * ldo + blk;
    for (int r = 0; r < c; ++r) X[(long long)r * ldo + c] = 0.0;
    X[(long long)c * ldo + c] = 1.0;
    for (int r = c + 1; r < NB; ++r) {
      double v = -T[r * LD + c];
      for (int t = c + 1; t < r; ++t) v = fma(-T[r * LD + t], X[(long long)t * ldo + c], v);
      X[(long long)r * ldo + c] = v;
    }
  } else {
    if (!Uinv) return;
    double* X = Uinv + blk * ldo + blk;
    for (int r = c + 1; r < NB; ++r) X[(long long)r * ldo + c] = 0.0;
    X[(long long)c * ldo + c] = 1.0 / T[c * LD + c];
    for (int r = c - 1; r >= 0; --r) {
      double v = 0.0;
      for (int t = r + 1; t <= c; ++t) v = fma(T[r * LD + t], X[(long long)t * ldo + c], v);
      X[(long long)r * ldo + c] = -v / T[r * LD + r];
    }
  }
}

void gemm(cudaStream_t st, int M, int N, int K, double alpha, const double* A, int lda, long long sA, const double* B, int ldb, long long sB,
          double beta, double* C, int ldc, long long sC, int batch, bool tri = false, const int* col_map = nullptr) {
  B200_CUDA(dtc::dgemm(st, M, N, K, alpha, A, lda, sA, B, ldb, sB, beta, C, ldc, sC, batch, tri, col_map));
  count_launch();
}

// A^-1 into A (n_pad x n_pad, row-major); W: 2 n_pad^2 doubles.  Returns 0, or the 1-based column of the first exactly zero
// pivot (A then holds the partial factors).
int lu_inverse(double* A, int n_pad, double* W, cudaStream_t st) {
  const int nblk = n_pad / NB;
  const long long nn = (long long)n_pad * n_pad;
  int per_sm = 0, dev = 0, sms = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, panel_getrf_kernel, PT, 0));
  const int max_grid = std::min(PT, std::max(1, per_sm) * sms);
  DevBuf<int> ipiv((size_t)n_pad), perm((size_t)n_pad), info(1), cand_idx((size_t)2 * max_grid);
  DevBuf<double> cand_rows((size_t)2 * max_grid * NB), cand_val((size_t)2 * max_grid), diag_rows((size_t)2 * NB),
      l11inv((size_t)NB * NB), T((size_t)n_pad * NB);
  B200_CUDA(cudaMemsetAsync(info.get(), 0, sizeof(int), st));
  B200_CUDA(cudaFuncSetAttribute(tri_inv_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TRI_SMEM));
  // ---- 1. getrf
  for (int k = 0; k < nblk; ++k) {
    const int k0 = k * NB, rows = n_pad - k0, rem = rows - NB;
    double* Akk = A + (long long)k0 * n_pad + k0;
    int grid = std::min(max_grid, (int)div_up(rows, 64));
    int ld = n_pad;
    int* ip = ipiv.get() + k0;
    int* inf = info.get();
    double *cr = cand_rows.get(), *cv = cand_val.get(), *dr = diag_rows.get();
    int* ci = cand_idx.get();
    void* args[] = {&Akk, &ld, (void*)&rows, (void*)&k0, &ip, &inf, &cr, &cv, &ci, &dr};
    B200_CUDA(cudaLaunchCooperativeKernel((void*)panel_getrf_kernel, dim3(grid), dim3(PT), args, 0, st));
    count_launch();
    laswp_kernel<<<div_up(n_pad, 256), 256, 0, st>>>(A, n_pad, n_pad, k0, ipiv.get());
    count_launch();
    if (rem > 0) {
      tri_inv_blocks_kernel<<<1, 2 * NB, TRI_SMEM, st>>>(Akk, n_pad, l11inv.get(), nullptr, NB);
      count_launch();
      double* A12 = Akk + NB;
      double* A21 = Akk + (long long)NB * n_pad;
      gemm(st, NB, rem, NB, 1.0, l11inv.get(), NB, 0, A12, n_pad, 0, 0.0, A12, n_pad, 0, 1);  // U12 = inv(L11) A12
      gemm(st, rem, rem, NB, -1.0, A21, n_pad, 0, A12, n_pad, 0, 1.0, A21 + NB, n_pad, 0, 1);  // A22 -= L21 U12
    }
  }
  int h_info = 0;
  std::vector<int> h_ipiv((size_t)n_pad);
  B200_CUDA(cudaMemcpyAsync(&h_info, info.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(h_ipiv.data(), ipiv.get(), sizeof(int) * (size_t)n_pad, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (h_info != 0) return h_info;
  // ---- 2. getri: U^-1 (upper) in W, L^-1 (unit lower) in W + n_pad^2
  double* Uinv = W;
  double* Linv = W + nn;
  B200_CUDA(cudaMemsetAsync(W, 0, sizeof(double) * (size_t)(2 * nn), st));
  tri_inv_blocks_kernel<<<nblk, 2 * NB, TRI_SMEM, st>>>(A, n_pad, Linv, Uinv, n_pad);
  count_launch();
  const long long ds = (long long)NB * n_pad + NB, bb = (long long)NB * NB;  // block (k, k) -> (k+1, k+1); one T block
  for (int d = 1; d < nblk; ++d) {
    const int batch = nblk - d;
    // U^-1[k, k+d] = -U^-1[k, k] (U[k, k+1 .. k+d] U^-1[k+1 .. k+d, k+d])
    gemm(st, NB, NB, d * NB, 1.0, A + NB, n_pad, ds, Uinv + (long long)NB * n_pad + (long long)d * NB, n_pad, ds, 0.0, T.get(), NB, bb, batch);
    gemm(st, NB, NB, NB, -1.0, Uinv, n_pad, ds, T.get(), NB, bb, 0.0, Uinv + (long long)d * NB, n_pad, ds, batch);
    // L^-1[k+d, k] = -L^-1[k+d, k+d] (L[k+d, k .. k+d-1] L^-1[k .. k+d-1, k])
    gemm(st, NB, NB, d * NB, 1.0, A + (long long)d * NB * n_pad, n_pad, ds, Linv, n_pad, ds, 0.0, T.get(), NB, bb, batch);
    gemm(st, NB, NB, NB, -1.0, Linv + (long long)d * NB * n_pad + (long long)d * NB, n_pad, ds, T.get(), NB, bb, 0.0,
         Linv + (long long)d * NB * n_pad, n_pad, ds, batch);
  }
  // P A = L U with P the interchanges in order: row i of P A is row perm[i] of A, so column i of U^-1 L^-1 is column perm[i]
  // of A^-1
  std::vector<int> h_perm((size_t)n_pad);
  for (int i = 0; i < n_pad; ++i) h_perm[i] = i;
  for (int j = 0; j < n_pad; ++j) std::swap(h_perm[j], h_perm[h_ipiv[j]]);
  B200_CUDA(cudaMemcpyAsync(perm.get(), h_perm.data(), sizeof(int) * (size_t)n_pad, cudaMemcpyHostToDevice, st));
  gemm(st, n_pad, n_pad, n_pad, 1.0, Uinv, n_pad, 0, Linv, n_pad, 0, 0.0, A, n_pad, 0, 1, true, perm.get());
  B200_CUDA(cudaStreamSynchronize(st));  // h_perm is read by the copy above; the device buffers die with this frame
  return 0;
}

}  // namespace lu
}  // namespace b200

using namespace b200;

extern "C" {

int b200_lu_inverse_device(double* d_A, int n_pad, double* d_work, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_A && d_work && n_pad > 0 && n_pad % lu::NB == 0, "b200_lu_inverse: n_pad must be a positive multiple of %d", lu::NB);
    const int info = lu::lu_inverse(d_A, n_pad, d_work, (cudaStream_t)stream);
    if (info != 0) {
      set_error("b200_lu_inverse: singular matrix (zero pivot at column %d)", info - 1);
      throw CudaFail{B200_E_SINGULAR};
    }
  });
}

int b200_debug_dgemm_device(int kind, int M, int N, int K, double alpha, const double* d_A, int lda, const double* d_B, int ldb,
                            double beta, double* d_C, int ldc, void* stream) {
  return guarded([&] {
    B200_REQUIRE(kind >= 0 && kind <= 2, "b200_debug_dgemm: kind must be 0, 1 or 2");
    B200_REQUIRE(d_A && d_B && d_C && M > 0 && N > 0 && K > 0 && M % 128 == 0 && N % 128 == 0 && K % 16 == 0,
                 "b200_debug_dgemm: M, N must be multiples of 128 and K of 16");
    B200_REQUIRE(lda % 2 == 0 && ldb % 2 == 0 && ldc % 2 == 0 && lda >= K && ldb >= N && ldc >= N &&
                     ((uintptr_t)d_A | (uintptr_t)d_B | (uintptr_t)d_C) % 16 == 0,
                 "b200_debug_dgemm: leading dimensions must be even and cover the matrix, pointers 16-byte aligned");
    B200_REQUIRE(kind != 2 || (M == K && N == K), "b200_debug_dgemm: kind 2 needs M == N == K");
    cudaStream_t st = (cudaStream_t)stream;
    if (kind == 0) lu::gemm(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
    else if (kind == 1)
      lu::gemm(st, 128, N, K, alpha, d_A, lda, 128LL * lda, d_B, ldb, (long long)K * ldb, beta, d_C, ldc, 128LL * ldc, M / 128);
    else lu::gemm(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1, true);
    B200_CUDA(cudaStreamSynchronize(st));
  });
}

}  // extern "C"
