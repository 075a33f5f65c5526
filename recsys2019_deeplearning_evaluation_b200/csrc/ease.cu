// K5: EASE^R closed form on the device, sm_90a.
//
// Replaces EASE_R/EASE_R_Recommender.py:55-69:  G = X^T X (through Compute_Similarity, shrink 0, normalize False,
// topK = n_items), G[diag] = item_popularity + l2_norm (nnz count per column, :62-63), P = inv(G) (np.linalg.inv on
// float32 -> LAPACK sgetrf/sgetri), B = P / (-diag P) (column j divided by -P_jj), B[diag] = 0.
//
// The Gram matrix comes from the dense mode of the similarity kernel (csrc/sim_topk.cu).  G is symmetric positive
// definite (l2_norm > 0), so the inverse is formed through a blocked Cholesky factorisation instead of LU:
//   1. right-looking blocked Cholesky, NB = 128: diagonal block factor + its inverse in one CTA (shared memory),
//      panel L21 = A21 inv(L11)^T and trailing update A22 -= L21 L21^T as GEMMs;
//   2. inverse of the factor block column by block column, one batched GEMM pair per block diagonal;
//   3. P = Linv^T Linv with the K range of every tile clipped to the non-zero (lower-triangular) part.
// All three are O(n^3) GEMM work and run on the tensor cores: gemm_tc2.cuh / gemm_tc.cuh (wgmma .tf32 with a 3xTF32 operand
// split for fp32-level accuracy -- the reference inverts in fp32 LAPACK -- accumulators in registers).  Only the 128 x 128
// diagonal-block factorisations stay on the CUDA cores (one CTA each, O(n * NB^2) work in total).
#include <algorithm>
#include <vector>

#include <stdlib.h>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "gemm_tc2.cuh"

namespace b200 {
namespace ease {

constexpr int NB = 128;  // Cholesky block size == GEMM tile size

// Cholesky of the NB x NB diagonal block at A (row-major, lda) in place (lower triangle; the strict upper triangle is
// zeroed) and its inverse into Inv (NB x NB, dense row-major, upper part zero).  One CTA, the block lives in smem.
__global__ void __launch_bounds__(256) potrf_inv_block_kernel(float* A, int lda, float* Inv, int* info) {
  extern __shared__ float L[];  // NB x (NB + 1)
  const int tid = threadIdx.x;
  constexpr int LD = NB + 1;
  for (int e = tid; e < NB * NB; e += 256) { const int r = e / NB, c = e % NB; L[r * LD + c] = A[(long long)r * lda + c]; }
  __syncthreads();
  for (int j = 0; j < NB; ++j) {
    if (tid == 0) {
      const float d = L[j * LD + j];
      if (!(d > 0.f)) atomicExch(info, j + 1);
      L[j * LD + j] = sqrtf(fmaxf(d, 1e-30f));
    }
    __syncthreads();
    const float djj = L[j * LD + j];
    for (int r = j + 1 + tid; r < NB; r += 256) L[r * LD + j] /= djj;
    __syncthreads();
    // trailing update of the lower triangle: L[r][c] -= L[r][j] * L[c][j] for j < c <= r
    const int rem = NB - j - 1;
    for (int e = tid; e < rem * rem; e += 256) {
      const int r = j + 1 + e / rem, c = j + 1 + e % rem;
      if (c <= r) L[r * LD + c] -= L[r * LD + j] * L[c * LD + j];
    }
    __syncthreads();
  }
  for (int e = tid; e < NB * NB; e += 256) { const int r = e / NB, c = e % NB; A[(long long)r * lda + c] = c <= r ? L[r * LD + c] : 0.f; }
  // inverse by forward substitution, one column per thread: X[:, c] solves L x = e_c
  for (int c = tid; c < NB; c += 256) {
    for (int r = 0; r < NB; ++r) {
      float v = (r == c) ? 1.f : 0.f;
      if (r >= c) {
        for (int t = c; t < r; ++t) v -= L[r * LD + t] * Inv[(long long)t * NB + c];
        v /= L[r * LD + r];
      } else {
        v = 0.f;
      }
      Inv[(long long)r * NB + c] = v;
    }
  }
}

__global__ void set_diag_kernel(float* G, int n, int n_pad, const int* __restrict__ csc_cnt, float l2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pad) return;
  G[(long long)j * n_pad + j] = j < n ? (float)csc_cnt[j] + l2 : 1.0f;  // EASE_R_Recommender.py:62-63; identity on the padding
}

__global__ void col_count_kernel(const int* __restrict__ idx, long long nnz, int* cnt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(cnt + idx[i], 1);
}

// B[i, j] = P[i, j] / (-P[j, j]), B[j, j] = 0 (EASE_R_Recommender.py:67-69); P padded (ldp), B compact n x n
__global__ void ease_finish_kernel(const float* __restrict__ P, int ldp, int n, float* Bout) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n * n) return;
  const int i = (int)(g / n), j = (int)(g % n);
  Bout[g] = i == j ? 0.f : P[(long long)i * ldp + j] / (-P[(long long)j * ldp + j]);
}

__global__ void copy_block_kernel(const float* __restrict__ src, int lds, float* dst, int ldd, int rows, int cols) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)rows * cols) return;
  const int r = (int)(g / cols), c = (int)(g % cols);
  dst[(long long)r * ldd + c] = src[(long long)r * lds + c];
}

// 2 = gemm_tc2.cuh (default: packed operands + cp.async.bulk producer), 1 = gemm_tc.cuh (the first kernel, kept selectable
// with B200REC_GEMM=1 for A/B timing)
int g_gemm_version = -1;
int gemm_version() {
  if (g_gemm_version < 0) {
    const char* e = getenv("B200REC_GEMM");
    g_gemm_version = (e && atoi(e) == 1) ? 1 : 2;
  }
  return g_gemm_version;
}

DevBuf<float> g_pack_a, g_pack_b;  // packed-operand workspaces of the v2 path, grown on demand

template <bool TA, bool TB, bool TRI>
void gemm_v2(cudaStream_t st, int M, int N, int K, float alpha, const float* A, int lda, long long sA, const float* B, int ldb,
             long long sB, float beta, float* C, int ldc, long long sC, int batch) {
  const int KC = K / tc::BK, RA = M / tc::BM, RB = N / tc::BN;
  const long long strideAp = (long long)RA * KC * tc2::PAIR_FLOATS, strideBp = (long long)RB * KC * tc2::PAIR_FLOATS;
  // op(A) and op(B) are the same memory pattern of the same matrix (L21 L21^T, Linv^T Linv): pack once
  const bool share = (A == B && lda == ldb && sA == sB && M == N && ((!TA) == TB));
  const size_t needA = (size_t)batch * (size_t)strideAp, needB = share ? 0 : (size_t)batch * (size_t)strideBp;
  if (g_pack_a.n < needA || g_pack_b.n < needB) {
    B200_CUDA(cudaStreamSynchronize(st));  // earlier kernels may still read the old workspaces
    if (g_pack_a.n < needA) g_pack_a.alloc(needA);
    if (g_pack_b.n < needB) g_pack_b.alloc(needB);
  }
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(tc2::tc2_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc2::SMEM_BYTES));
    configured = true;
  }
  tc2::pack_tiles_kernel<!TA><<<dim3(KC, RA, batch), tc2::THREADS, 2 * tc::TILE_BYTES, st>>>(A, lda, sA, g_pack_a.get(), strideAp);
  count_launch();
  if (!share) {
    tc2::pack_tiles_kernel<TB><<<dim3(KC, RB, batch), tc2::THREADS, 2 * tc::TILE_BYTES, st>>>(B, ldb, sB, g_pack_b.get(), strideBp);
    count_launch();
  }
  tc2::tc2_gemm_kernel<<<dim3(RB, RA, batch), tc2::GEMM_THREADS, tc2::SMEM_BYTES, st>>>(
      K, TRI ? 1 : 0, alpha, g_pack_a.get(), strideAp, share ? g_pack_a.get() : g_pack_b.get(), share ? strideAp : strideBp, beta, C, ldc, sC);
  count_launch();
}

template <bool TA, bool TB, bool TRI>
void gemm(cudaStream_t st, int M, int N, int K, float alpha, const float* A, int lda, long long sA, const float* B, int ldb,
          long long sB, float beta, float* C, int ldc, long long sC, int batch) {
  if (M <= 0 || N <= 0 || batch <= 0) return;
  if (gemm_version() == 2) {
    gemm_v2<TA, TB, TRI>(st, M, N, K, alpha, A, lda, sA, B, ldb, sB, beta, C, ldc, sC, batch);
    return;
  }
  static bool configured = false;
  if (!configured) {
    B200_CUDA(cudaFuncSetAttribute(tc::tc_gemm_kernel<TA, TB, TRI>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
    configured = true;
  }
  tc::tc_gemm_kernel<TA, TB, TRI><<<dim3(N / tc::BN, M / tc::BM, batch), tc::THREADS, tc::SMEM_BYTES, st>>>(
      M, N, K, alpha, A, lda, sA, B, ldb, sB, beta, C, ldc, sC);
  count_launch();
}

}  // namespace ease
}  // namespace b200

using namespace b200;
using namespace b200::ease;

extern "C" {

// In-place inverse of a symmetric positive definite n_pad x n_pad matrix (n_pad multiple of 128, row-major, device).
// On return d_A holds A^{-1} (full symmetric matrix).  d_work: 2 * n_pad * n_pad floats.
int b200_spd_inverse_device(float* d_A, int n_pad, float* d_work, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_A && d_work && n_pad > 0 && n_pad % NB == 0, "b200_spd_inverse: n_pad must be a positive multiple of %d", NB);
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = n_pad / NB;
    const long long nn = (long long)n_pad * n_pad;
    float* Linv = d_work;        // n_pad x n_pad
    float* panel = d_work + nn;  // n_pad x NB  (first part of the second workspace)
    DevBuf<float> inv_blocks((size_t)nblk * NB * NB);
    DevBuf<int> info(1);
    B200_CUDA(cudaMemsetAsync(info.get(), 0, sizeof(int), st));
    B200_CUDA(cudaFuncSetAttribute(potrf_inv_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, NB * (NB + 1) * 4));
    // ---- 1. blocked Cholesky (lower), A = L L^T
    for (int k = 0; k < nblk; ++k) {
      float* Akk = d_A + (long long)k * NB * n_pad + (long long)k * NB;
      potrf_inv_block_kernel<<<1, 256, NB * (NB + 1) * 4, st>>>(Akk, n_pad, inv_blocks.get() + (size_t)k * NB * NB, info.get());
      count_launch();
      const int rem = n_pad - (k + 1) * NB;
      if (rem > 0) {
        float* A21 = Akk + (long long)NB * n_pad;
        // panel = A21 * inv(L11)^T
        gemm<false, true, false>(st, rem, NB, NB, 1.f, A21, n_pad, 0, inv_blocks.get() + (size_t)k * NB * NB, NB, 0, 0.f, panel, NB, 0, 1);
        copy_block_kernel<<<div_up((long long)rem * NB, 256), 256, 0, st>>>(panel, NB, A21, n_pad, rem, NB);
        count_launch();
        // A22 -= L21 * L21^T
        float* A22 = A21 + NB;
        gemm<false, true, false>(st, rem, rem, NB, -1.f, A21, n_pad, 0, A21, n_pad, 0, 1.f, A22, n_pad, 0, 1);
      }
    }
    int h_info = 0;
    B200_CUDA(cudaMemcpyAsync(&h_info, info.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_REQUIRE(h_info == 0, "b200_spd_inverse: matrix is not positive definite (pivot %d of a diagonal block)", h_info);
    // ---- 2. Linv = L^{-1}: diagonal blocks, then one block diagonal at a time
    B200_CUDA(cudaMemsetAsync(Linv, 0, sizeof(float) * (size_t)nn, st));
    for (int k = 0; k < nblk; ++k) {
      copy_block_kernel<<<div_up((long long)NB * NB, 256), 256, 0, st>>>(inv_blocks.get() + (size_t)k * NB * NB, NB,
                                                                         Linv + (long long)k * NB * n_pad + (long long)k * NB, n_pad, NB, NB);
    }
    count_launch(nblk);
    const long long diag_stride = (long long)NB * n_pad + NB;  // from block (k, k) to block (k+1, k+1)
    float* T = panel;                                          // nblk blocks of NB x NB
    for (int d = 1; d < nblk; ++d) {
      const int batch = nblk - d;
      // T_k = L[k+d, k .. k+d-1] * Linv[k .. k+d-1, k]      (NB x d*NB) * (d*NB x NB)
      gemm<false, false, false>(st, NB, NB, d * NB, 1.f, d_A + (long long)d * NB * n_pad, n_pad, diag_stride, Linv, n_pad, diag_stride, 0.f,
                                T, NB, (long long)NB * NB, batch);
      // Linv[k+d, k] = -inv(L[k+d, k+d]) * T_k
      gemm<false, false, false>(st, NB, NB, NB, -1.f, inv_blocks.get() + (size_t)d * NB * NB, NB, (long long)NB * NB, T, NB,
                                (long long)NB * NB, 0.f, Linv + (long long)d * NB * n_pad, n_pad, diag_stride, batch);
    }
    // ---- 3. A^{-1} = Linv^T * Linv  (k >= max(i, j) only)
    gemm<true, false, true>(st, n_pad, n_pad, n_pad, 1.f, Linv, n_pad, 0, Linv, n_pad, 0, 0.f, d_A, n_pad, 0, 1);
    B200_CUDA(cudaGetLastError());
  });
}

// TEST HOOK: one GEMM of the blocked inverse through version 1 (gemm_tc.cuh) or 2 (gemm_tc2.cuh):
//   kind 0: C = alpha A B^T + beta C   (A [M,K] row-major, B [N,K] row-major)        -- panel / trailing updates
//   kind 1: C = alpha A B + beta C     (A [M,K] row-major, B [K,N] row-major)        -- factor-inverse blocks
//   kind 2: C = alpha A^T B + beta C restricted to k >= max(row block, column block) (A [K,M], B [K,N]) -- Linv^T Linv
// M, N multiples of 128, K a multiple of 32; all pointers on the device.
int b200_debug_gemm_device(int version, int kind, int M, int N, int K, float alpha, const float* d_A, int lda, const float* d_B,
                           int ldb, float beta, float* d_C, int ldc, void* stream) {
  return guarded([&] {
    B200_REQUIRE(version == 1 || version == 2, "b200_debug_gemm: version must be 1 or 2");
    B200_REQUIRE(kind >= 0 && kind <= 2, "b200_debug_gemm: kind must be 0, 1 or 2");
    B200_REQUIRE(d_A && d_B && d_C && M > 0 && N > 0 && K > 0 && M % 128 == 0 && N % 128 == 0 && K % 32 == 0,
                 "b200_debug_gemm: M, N must be multiples of 128 and K of 32");
    cudaStream_t st = (cudaStream_t)stream;
    const int saved = gemm_version();
    g_gemm_version = version;
    try {
      if (kind == 0) gemm<false, true, false>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
      else if (kind == 1) gemm<false, false, false>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
      else gemm<true, false, true>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
      B200_CUDA(cudaGetLastError());
      B200_CUDA(cudaStreamSynchronize(st));
    } catch (...) {
      g_gemm_version = saved;
      throw;
    }
    g_gemm_version = saved;
  });
}

/* EASE_R fit from a precomputed dense Gram block: d_G is [n_items, n_items] row-major holding X^T X off the diagonal
 * (the dense mode of the similarity kernel).  Writes B (n_items x n_items, fp32) to h_B (host) and/or d_B (device). */
int b200_ease_from_gram_device(const float* d_G, int n_items, const int32_t* d_urm_indices, int64_t nnz, float l2_norm, float* h_B,
                               float* d_B, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_G && n_items > 0 && (h_B || d_B), "b200_ease_from_gram: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int n = n_items, n_pad = ((n + NB - 1) / NB) * NB;
    const long long nn = (long long)n_pad * n_pad;
    DevBuf<float> A((size_t)nn), work((size_t)2 * nn);
    DevBuf<int> cnt((size_t)n);
    B200_CUDA(cudaMemsetAsync(A.get(), 0, sizeof(float) * (size_t)nn, st));
    B200_CUDA(cudaMemsetAsync(cnt.get(), 0, sizeof(int) * (size_t)n, st));
    copy_block_kernel<<<div_up((long long)n * n, 256), 256, 0, st>>>(d_G, n, A.get(), n_pad, n, n);
    count_launch();
    if (nnz > 0) { col_count_kernel<<<sm_count() * 8, 256, 0, st>>>(d_urm_indices, nnz, cnt.get()); count_launch(); }
    set_diag_kernel<<<div_up(n_pad, 256), 256, 0, st>>>(A.get(), n, n_pad, cnt.get(), l2_norm);
    count_launch();
    int rc = b200_spd_inverse_device(A.get(), n_pad, work.get(), stream);
    if (rc != B200_OK) throw CudaFail{rc};
    DevBuf<float> tmpB;
    float* out = d_B;
    if (!out) { tmpB.alloc((size_t)n * n); out = tmpB.get(); }
    ease_finish_kernel<<<div_up((long long)n * n, 256), 256, 0, st>>>(A.get(), n_pad, n, out);
    count_launch();
    B200_CUDA(cudaGetLastError());
    if (h_B) B200_CUDA(cudaMemcpyAsync(h_B, out, sizeof(float) * (size_t)n * n, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  });
}

}  // extern "C"
