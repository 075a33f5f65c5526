// K5: EASE^R closed form on the device, sm_90a.
//
// Replaces EASE_R/EASE_R_Recommender.py:55-69:  G = X^T X (through Compute_Similarity, shrink 0, normalize False,
// topK = n_items), G[diag] = item_popularity + l2_norm (nnz count per column, :62-63), P = inv(G) (np.linalg.inv on
// float32: LAPACK dgetrf/dgetri in float64, rounded to float32), B = P / (-diag P) (column j divided by -P_jj), B[diag] = 0.
//
// The Gram matrix comes from the dense mode of the similarity kernel (csrc/sim_topk.cu).  When G is symmetric positive
// definite (binary data, or a large enough l2_norm) the inverse is formed through a blocked Cholesky factorisation:
//   1. right-looking blocked Cholesky, NB = 128: diagonal block factor + its inverse in one CTA (shared memory),
//      panel L21 = A21 inv(L11)^T and trailing update A22 -= L21 L21^T as GEMMs;
//   2. inverse of the factor block column by block column, one batched GEMM pair per block diagonal;
//   3. P = Linv^T Linv with the K range of every tile clipped to the non-zero (lower-triangular) part.
// All three are O(n^3) GEMM work and run on the tensor cores: gemm_tc2.cuh (wgmma .tf32 with a 3xTF32 operand split for
// fp32-level accuracy, accumulators in registers).  Only the 128 x 128 diagonal-block factorisations stay on the
// CUDA cores (one CTA each, O(n * NB^2) work in total).
// The popularity diagonal is a count, below sum r^2 on explicit ratings, so there G can be indefinite.  When the Cholesky
// meets a non-positive pivot, G is inverted again in fp64 by the pivoted LU of lu_inverse.cu (what np.linalg.inv does);
// an fp32 LU of these systems (cond up to ~1e7) would be far from the reference.
// Catalogues whose footprint here (G, B and 5 n_pad^2 floats) does not fit take b200_ease_inplace_device: the same
// Cholesky, then trtri and lauum in place and an in-place finish, all inside one n_pad^2 buffer (no LU fallback there).
#include <algorithm>
#include <vector>

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

// fp64 copy of G padded to n_pad with the diagonal set_diag_kernel writes (the fp32 values, widened): input of the LU path
__global__ void widen_gram_kernel(const float* __restrict__ G, int n, int n_pad, const int* __restrict__ csc_cnt, float l2, double* A) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_pad * n_pad) return;
  const int i = (int)(g / n_pad), j = (int)(g % n_pad);
  float v = i == j ? 1.0f : 0.0f;
  if (i < n && j < n) v = i == j ? (float)csc_cnt[j] + l2 : G[(long long)i * n + j];
  A[g] = (double)v;
}

// ease_finish_kernel on the fp64 inverse: the quotient in fp64, rounded once to fp32
__global__ void ease_finish64_kernel(const double* __restrict__ P, int ldp, int n, float* Bout) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n * n) return;
  const int i = (int)(g / n), j = (int)(g % n);
  Bout[g] = i == j ? 0.f : (float)(P[(long long)i * ldp + j] / (-P[(long long)j * ldp + j]));
}

__global__ void copy_block_kernel(const float* __restrict__ src, int lds, float* dst, int ldd, int rows, int cols) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)rows * cols) return;
  const int r = (int)(g / cols), c = (int)(g % cols);
  dst[(long long)r * ldd + c] = src[(long long)r * lds + c];
}

DevBuf<float> g_pack_a, g_pack_b;  // packed-operand workspaces of gemm, grown on demand

// C = alpha op(A) op(B) + beta C through gemm_tc2.cuh: pack op(A) and op(B) into the workspaces, then the GEMM kernel.
// TA: op(A)(m, k) = A[k * lda + m]; TB: op(B)(k, n) = B[n * ldb + k].  TRI: op(A) = L^T, op(B) = L with L lower
// triangular, so only k >= max(m0, n0) contributes.  M, N multiples of 128, K a multiple of 32.
template <bool TA, bool TB, bool TRI>
void gemm(cudaStream_t st, int M, int N, int K, float alpha, const float* A, int lda, long long sA, const float* B, int ldb,
          long long sB, float beta, float* C, int ldc, long long sC, int batch) {
  if (M <= 0 || N <= 0 || batch <= 0) return;
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

// 1. Right-looking blocked Cholesky (lower) of the n_pad x n_pad matrix at d_A in place, A = L L^T: every diagonal block is
// factored (strict upper triangle zeroed) and its inverse written to inv_blocks (n_pad / NB blocks of NB x NB); the blocks
// above the diagonal keep their stale input values.  panel: n_pad x NB floats.  Returns 0, or the 1-based position of the
// first non-positive pivot inside a diagonal block (the factorisation runs to the end).
int cholesky(float* d_A, int n_pad, float* inv_blocks, float* panel, cudaStream_t st) {
  const int nblk = n_pad / NB;
  DevBuf<int> info(1);
  B200_CUDA(cudaMemsetAsync(info.get(), 0, sizeof(int), st));
  B200_CUDA(cudaFuncSetAttribute(potrf_inv_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, NB * (NB + 1) * 4));
  for (int k = 0; k < nblk; ++k) {
    float* Akk = d_A + (long long)k * NB * n_pad + (long long)k * NB;
    potrf_inv_block_kernel<<<1, 256, NB * (NB + 1) * 4, st>>>(Akk, n_pad, inv_blocks + (size_t)k * NB * NB, info.get());
    count_launch();
    const int rem = n_pad - (k + 1) * NB;
    if (rem > 0) {
      float* A21 = Akk + (long long)NB * n_pad;
      // panel = A21 * inv(L11)^T
      gemm<false, true, false>(st, rem, NB, NB, 1.f, A21, n_pad, 0, inv_blocks + (size_t)k * NB * NB, NB, 0, 0.f, panel, NB, 0, 1);
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
  return h_info;
}

// In-place inverse of a symmetric positive definite n_pad x n_pad matrix (n_pad multiple of 128, row-major, device).
// Returns 0 with A^{-1} (full symmetric matrix) in d_A, or the 1-based position of the first non-positive pivot inside a
// diagonal block (the factorisation runs to the end, no inverse is formed).  d_work: 2 * n_pad * n_pad floats.
int spd_inverse(float* d_A, int n_pad, float* d_work, cudaStream_t st) {
  const int nblk = n_pad / NB;
  const long long nn = (long long)n_pad * n_pad;
  float* Linv = d_work;        // n_pad x n_pad
  float* panel = d_work + nn;  // n_pad x NB  (first part of the second workspace)
  DevBuf<float> inv_blocks((size_t)nblk * NB * NB);
  const int h_info = cholesky(d_A, n_pad, inv_blocks.get(), panel, st);
  if (h_info != 0) return h_info;
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
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// In-place EASE fit: the whole inverse and the finish inside the one n_pad x n_pad buffer (LAPACK potrf -> trtri -> lauum).
// The only O(n^3) products with a K range of more than NB are split into K chunks of KW, so the packed operands of gemm
// stay at 2 * n_pad * KW floats each instead of growing with n_pad^2.
constexpr int KW = 4 * NB;

// A[r, c] = 0 for c > r: the blocks above the diagonal still hold G after cholesky(), and the K-chunked trtri products
// read the part of them inside a chunk (which must be the zeros of the triangular factor).  One CTA per row.
__global__ void zero_upper_kernel(float* A, int n_pad) {
  const long long r = blockIdx.x;
  for (int c = (int)r + 1 + threadIdx.x; c < n_pad; c += blockDim.x) A[r * n_pad + c] = 0.f;
}

__global__ void zero_block_kernel(float* dst, int ldd, int rows, int cols) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)rows * cols) return;
  dst[(g / cols) * ldd + g % cols] = 0.f;
}

__global__ void get_diag_kernel(const float* __restrict__ A, int ldp, int n, float* d) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) d[j] = A[(long long)j * ldp + j];
}

// In-place EASE finish on the lower triangle of P (stride ldp), d = diag P saved beforehand: B[i, j] = P[i, j] / (-d[j]),
// B[j, j] = 0.  One CTA owns the 32 x 32 tile pair (I, J), (J, I) with I >= J: it reads the lower-triangle values of
// tile (I, J) into shared memory, then writes both tiles (P symmetric: P[j, i] = P[i, j]).  No CTA reads a tile another
// CTA writes.  grid = (T, T), T = ceil(n / 32); the CTAs with J > I exit.
__global__ void __launch_bounds__(256) ease_finish_inplace_kernel(float* A, int ldp, int n, const float* __restrict__ d) {
  __shared__ float t[32][33];
  const int I = blockIdx.y, J = blockIdx.x;
  if (J > I) return;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int r = ty; r < 32; r += 8) {
    const int i = I * 32 + r, j = J * 32 + tx;
    t[r][tx] = (i < n && j < n && i >= j) ? A[(long long)i * ldp + j] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    {  // tile (I, J)
      const int i = I * 32 + r, j = J * 32 + tx;
      if (i < n && j < n) A[(long long)i * ldp + j] = i == j ? 0.f : (i > j ? t[r][tx] : t[tx][r]) / (-d[j]);
    }
    if (I != J) {  // tile (J, I): P[i, j] = P[j, i] = t[tx][r]
      const int i = J * 32 + r, j = I * 32 + tx;
      if (i < n && j < n) A[(long long)i * ldp + j] = t[tx][r] / (-d[j]);
    }
  }
}

// 2. L := L^{-1} in place (LAPACK trtri, lower, non-unit), block columns right to left: X21 = -X22 L21 X11 with
// X11 = inv_blocks[j] and X22 (the trailing block, already inverted) read in K chunks of KW.  The strict upper triangle
// must be zero (zero_upper_kernel).  panel: n_pad x NB.
void trtri_inplace(float* d_A, int n_pad, const float* inv_blocks, float* panel, cudaStream_t st) {
  const int nblk = n_pad / NB;
  for (int k = 0; k < nblk; ++k)  // the diagonal blocks become X_kk; the L_kk values are not read again
    copy_block_kernel<<<div_up((long long)NB * NB, 256), 256, 0, st>>>(inv_blocks + (size_t)k * NB * NB, NB,
                                                                       d_A + (long long)k * NB * n_pad + (long long)k * NB, n_pad, NB, NB);
  count_launch(nblk);
  for (int j = nblk - 2; j >= 0; --j) {
    const int r0 = (j + 1) * NB, rem = n_pad - r0;
    float* A21 = d_A + (long long)r0 * n_pad + (long long)j * NB;
    // panel = L21 X11
    gemm<false, false, false>(st, rem, NB, NB, 1.f, A21, n_pad, 0, inv_blocks + (size_t)j * NB * NB, NB, 0, 0.f, panel, NB, 0, 1);
    // X21 = -X22 panel: the chunk of columns [k0, k0 + kw) of X22 only reaches rows >= k0 (X22 is lower triangular)
    for (int k0 = r0; k0 < n_pad; k0 += KW) {
      const int kw = std::min(KW, n_pad - k0);
      gemm<false, false, false>(st, n_pad - k0, NB, kw, -1.f, d_A + (long long)k0 * n_pad + k0, n_pad, 0,
                                panel + (long long)(k0 - r0) * NB, NB, 0, k0 == r0 ? 0.f : 1.f,
                                d_A + (long long)k0 * n_pad + (long long)j * NB, n_pad, 0, 1);
    }
  }
}

// 3. P := X^T X in place on the lower triangle (LAPACK lauum), block rows top to bottom: for block row i,
// A(i, 0:i+1) = X_ii^T A(i, 0:i+1) + X(i+1:, i)^T X(i+1:, 0:i+1).  The rows below i still hold X when row i is formed,
// and the first product packs its operands before it overwrites them.  The blocks above the diagonal are not written
// except the upper half of the diagonal blocks; only the lower triangle of P is meaningful.
void lauum_inplace(float* d_A, int n_pad, cudaStream_t st) {
  const int nblk = n_pad / NB;
  for (int i = 0; i < nblk; ++i) {
    const int N = (i + 1) * NB;
    float* Ai0 = d_A + (long long)i * NB * n_pad;
    gemm<true, false, false>(st, NB, N, NB, 1.f, Ai0 + (long long)i * NB, n_pad, 0, Ai0, n_pad, 0, 0.f, Ai0, n_pad, 0, 1);
    for (int k0 = (i + 1) * NB; k0 < n_pad; k0 += KW) {
      const int kw = std::min(KW, n_pad - k0);
      const float* Ak0 = d_A + (long long)k0 * n_pad;
      gemm<true, false, false>(st, NB, N, kw, 1.f, Ak0 + (long long)i * NB, n_pad, 0, Ak0, n_pad, 0, 1.f, Ai0, n_pad, 0, 1);
    }
  }
}

// Device bytes ease_inplace allocates besides the matrix: inv_blocks + panel, the packed operands of gemm (at most
// 2 * n_pad * min(KW, n_pad) floats each), popularity counts, diag P, the compaction stage (NB rows of n) and the pivot flag.
long long ease_inplace_workspace(int n) {
  const long long n_pad = ((n + NB - 1) / NB) * (long long)NB;
  return 4 * (2 * n_pad * NB + 2 * 2 * n_pad * std::min<long long>(KW, n_pad) + 2 * (long long)n + (long long)NB * n) + 4;
}

// Stages of ease_inplace on an SPD n_pad x n_pad matrix: 0 the Cholesky factor, 1 + L^{-1}, 2 + P = L^{-T} L^{-1}.
// Returns the pivot position of cholesky() (0 when positive definite; later stages are skipped otherwise).
int inverse_inplace(float* d_A, int n_pad, int last_stage, cudaStream_t st) {
  DevBuf<float> inv_blocks((size_t)n_pad * NB), panel((size_t)n_pad * NB);
  // the largest packed operand of the stages (K = NB, or a K chunk of at most min(KW, n_pad)): grow the workspaces once
  const size_t pack = (size_t)2 * n_pad * std::min(KW, n_pad);
  if (g_pack_a.n < pack || g_pack_b.n < pack) {
    B200_CUDA(cudaStreamSynchronize(st));
    if (g_pack_a.n < pack) g_pack_a.alloc(pack);
    if (g_pack_b.n < pack) g_pack_b.alloc(pack);
  }
  const int info = cholesky(d_A, n_pad, inv_blocks.get(), panel.get(), st);
  if (info != 0 || last_stage < 1) return info;
  zero_upper_kernel<<<n_pad, 256, 0, st>>>(d_A, n_pad);
  count_launch();
  trtri_inplace(d_A, n_pad, inv_blocks.get(), panel.get(), st);
  if (last_stage >= 2) lauum_inplace(d_A, n_pad, st);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaStreamSynchronize(st));  // inv_blocks and panel are freed on return
  return 0;
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
    const int info = spd_inverse(d_A, n_pad, d_work, (cudaStream_t)stream);
    B200_REQUIRE(info == 0, "b200_spd_inverse: matrix is not positive definite (pivot %d of a diagonal block)", info);
  });
}

// TEST HOOK: one GEMM of the blocked inverse (gemm_tc2.cuh):
//   kind 0: C = alpha A B^T + beta C   (A [M,K] row-major, B [N,K] row-major)        -- panel / trailing updates
//   kind 1: C = alpha A B + beta C     (A [M,K] row-major, B [K,N] row-major)        -- factor-inverse blocks
//   kind 2: C = alpha A^T B + beta C restricted to k >= max(row block, column block) (A [K,M], B [K,N]) -- Linv^T Linv
// M, N multiples of 128, K a multiple of 32; all pointers on the device.
int b200_debug_gemm_device(int kind, int M, int N, int K, float alpha, const float* d_A, int lda, const float* d_B, int ldb,
                           float beta, float* d_C, int ldc, void* stream) {
  return guarded([&] {
    B200_REQUIRE(kind >= 0 && kind <= 2, "b200_debug_gemm: kind must be 0, 1 or 2");
    B200_REQUIRE(d_A && d_B && d_C && M > 0 && N > 0 && K > 0 && M % 128 == 0 && N % 128 == 0 && K % 32 == 0,
                 "b200_debug_gemm: M, N must be multiples of 128 and K of 32");
    cudaStream_t st = (cudaStream_t)stream;
    if (kind == 0) gemm<false, true, false>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
    else if (kind == 1) gemm<false, false, false>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
    else gemm<true, false, true>(st, M, N, K, alpha, d_A, lda, 0, d_B, ldb, 0, beta, d_C, ldc, 0, 1);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(st));
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
    const bool spd = spd_inverse(A.get(), n_pad, work.get(), st) == 0;
    DevBuf<double> A64, work64;
    if (!spd) {
      // G + diag is not positive definite (explicit ratings: the popularity diagonal is below sum r^2): invert it as the
      // reference does, by LU with partial pivoting, in fp64 (np.linalg.inv computes in float64 for a float32 input)
      A.release();
      work.release();
      B200_CUDA(cudaStreamSynchronize(st));  // the Cholesky's GEMMs may still read the packed-operand workspaces
      g_pack_a.release();
      g_pack_b.release();
      A64.alloc((size_t)nn);
      work64.alloc((size_t)2 * nn);
      widen_gram_kernel<<<div_up(nn, 256), 256, 0, st>>>(d_G, n, n_pad, cnt.get(), l2_norm, A64.get());
      count_launch();
      const int rc = b200_lu_inverse_device(A64.get(), n_pad, work64.get(), stream);
      if (rc != B200_OK) throw CudaFail{rc};
      work64.release();
    }
    DevBuf<float> tmpB;
    float* out = d_B;
    if (!out) { tmpB.alloc((size_t)n * n); out = tmpB.get(); }
    if (spd) ease_finish_kernel<<<div_up((long long)n * n, 256), 256, 0, st>>>(A.get(), n_pad, n, out);
    else ease_finish64_kernel<<<div_up((long long)n * n, 256), 256, 0, st>>>(A64.get(), n_pad, n, out);
    count_launch();
    B200_CUDA(cudaGetLastError());
    if (h_B) B200_CUDA(cudaMemcpyAsync(h_B, out, sizeof(float) * (size_t)n * n, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  });
}

}  // extern "C"

extern "C" {

/* In-place EASE_R fit: d_A [n_pad, n_pad] fp32 (n_pad = n_items rounded up to 128) holds X^T X in its top-left
 * n_items x n_items block; on return its first n_items^2 floats are B as a contiguous [n_items, n_items] array. */
int b200_ease_inplace_device(float* d_A, int n_items, const int32_t* d_urm_indices, int64_t nnz, float l2_norm, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_A && n_items > 0 && (nnz == 0 || d_urm_indices), "b200_ease_inplace: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int n = n_items, n_pad = ((n + NB - 1) / NB) * NB;
    // identity padding: rows >= n and columns >= n are zero, then the diagonal (EASE_R_Recommender.py:62-63)
    if (n_pad > n) {
      zero_block_kernel<<<div_up((long long)n * (n_pad - n), 256), 256, 0, st>>>(d_A + n, n_pad, n, n_pad - n);
      count_launch();
      B200_CUDA(cudaMemsetAsync(d_A + (long long)n * n_pad, 0, sizeof(float) * (size_t)(n_pad - n) * n_pad, st));
    }
    {
      DevBuf<int> cnt((size_t)n);
      B200_CUDA(cudaMemsetAsync(cnt.get(), 0, sizeof(int) * (size_t)n, st));
      if (nnz > 0) { col_count_kernel<<<sm_count() * 8, 256, 0, st>>>(d_urm_indices, nnz, cnt.get()); count_launch(); }
      set_diag_kernel<<<div_up(n_pad, 256), 256, 0, st>>>(d_A, n, n_pad, cnt.get(), l2_norm);
      count_launch();
      B200_CUDA(cudaStreamSynchronize(st));
    }
    const int info = inverse_inplace(d_A, n_pad, 2, st);
    if (info != 0) {
      set_error("b200_ease_inplace: X^T X + diag is not positive definite (pivot %d of a diagonal block); the fp64 LU "
                "inverse needs %lld more device bytes", info, 24LL * n_pad * n_pad);
      throw CudaFail{B200_E_NOT_SPD};
    }
    {
      DevBuf<float> d((size_t)n);
      get_diag_kernel<<<div_up(n, 256), 256, 0, st>>>(d_A, n_pad, n, d.get());
      const unsigned T = div_up(n, 32);
      ease_finish_inplace_kernel<<<dim3(T, T), dim3(32, 8), 0, st>>>(d_A, n_pad, n, d.get());
      count_launch(2);
      B200_CUDA(cudaGetLastError());
      B200_CUDA(cudaStreamSynchronize(st));
    }
    if (n_pad > n) {
      // rows in order from stride n_pad to stride n through a stage of NB rows: the destination of rows [a, a + NB)
      // ends at (a + NB) n <= (a + NB) n_pad, where the sources not yet staged begin
      DevBuf<float> stage((size_t)NB * n);
      for (int a = 0; a < n; a += NB) {
        const int rows = std::min(NB, n - a);
        copy_block_kernel<<<div_up((long long)rows * n, 256), 256, 0, st>>>(d_A + (long long)a * n_pad, n_pad, stage.get(), n, rows, n);
        copy_block_kernel<<<div_up((long long)rows * n, 256), 256, 0, st>>>(stage.get(), n, d_A + (long long)a * n, n, rows, n);
        count_launch(2);
      }
      B200_CUDA(cudaGetLastError());
      B200_CUDA(cudaStreamSynchronize(st));
    }
  });
}

int b200_ease_inplace_workspace_bytes(int n_items, int64_t* bytes) {
  return guarded([&] {
    B200_REQUIRE(n_items > 0 && bytes, "b200_ease_inplace_workspace_bytes: n_items must be positive");
    *bytes = ease_inplace_workspace(n_items);
  });
}

/* TEST HOOK: the stages of the in-place inverse on an SPD [n_pad, n_pad] matrix (n_pad a multiple of 128):
 * op 0 the Cholesky factor, op 1 then L^{-1} (trtri), op 2 then P = L^{-T} L^{-1} (lauum). */
int b200_ease_inplace_debug_device(int op, float* d_A, int n_pad, void* stream) {
  return guarded([&] {
    B200_REQUIRE(op >= 0 && op <= 2 && d_A && n_pad > 0 && n_pad % NB == 0,
                 "b200_ease_inplace_debug: op must be 0, 1 or 2 and n_pad a positive multiple of %d", NB);
    const int info = inverse_inplace(d_A, n_pad, op, (cudaStream_t)stream);
    if (info != 0) {
      set_error("b200_ease_inplace_debug: matrix is not positive definite (pivot %d of a diagonal block)", info);
      throw CudaFail{B200_E_NOT_SPD};
    }
  });
}

}  // extern "C"
