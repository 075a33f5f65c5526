// fp64 tensor-core GEMM for the LU inverse (lu_inverse.cu), sm_90a: mma.sync m16n8k16 .f64 (DMMA.16x8x16), accumulators
// in registers.  Only the row-major NN shapes the blocked LU and its inverse need:
//   C = alpha A B + beta C                       A [M,K], B [K,N], C [M,N], all row-major with leading dimensions;
//   batched over blockIdx.z with element strides sA, sB, sC (the block-diagonal triangular inverses);
//   tri != 0: each 128 x 128 tile (bm, bn) sums only k >= max(bm, bn) * 128 (U^-1 L^-1 of two triangular factors);
//   col_map != nullptr: column j of the product is written to column col_map[j] of C (beta must be 0; the column
//   permutation of getri folded into the store).
// M, N multiples of 128, K a multiple of 16; lda, ldb, ldc even and A, B 16-byte aligned (cp.async 16-byte copies).
// Tile 128 x 128 x 16 per CTA, 8 warps as 2 (M) x 4 (N), 64 x 32 per warp; a 4-stage cp.async ring in shared memory.
#pragma once
#include <cuda_runtime.h>

namespace b200 {
namespace dtc {

constexpr int BM = 128, BN = 128, BK = 16, STAGES = 4, THREADS = 256;
constexpr int LDA_S = BK + 4;   // doubles; 8*row + 2*col (mod 32 banks): each bank pair is hit twice per warp, the 64-bit minimum
constexpr int LDB_S = BN + 4;   // doubles; 8*k + 2*col (mod 32 banks): same
constexpr int A_STAGE = BM * LDA_S, B_STAGE = BK * LDB_S;  // doubles
constexpr int SMEM_BYTES = STAGES * (A_STAGE + B_STAGE) * 8;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// D = A B + D, A 16 x 16 (a[i]: row g + 8 (i % 2), col t + 4 (i / 2)), B 16 x 8 (b[i]: row t + 4 i, col g),
// D 16 x 8 (d[0..1]: row g, cols 2t, 2t + 1; d[2..3]: row g + 8), g = lane / 4, t = lane % 4.
__device__ __forceinline__ void dmma16816(double* d, const double* a, const double* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};\n"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
        "d"(b[3]));
}

__global__ void __launch_bounds__(THREADS, 1)
    dgemm_kernel(int K, int tri, double alpha, const double* __restrict__ A, int lda, long long sA, const double* __restrict__ B,
                 int ldb, long long sB, double beta, double* C, int ldc, long long sC, const int* __restrict__ col_map) {
  extern __shared__ __align__(16) double smem[];
  double* As = smem;
  double* Bs = smem + STAGES * A_STAGE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 2) * 64, wn = (warp & 3) * 32;
  const int bm = blockIdx.y, bn = blockIdx.x;
  A += (long long)blockIdx.z * sA + (long long)bm * BM * lda;
  B += (long long)blockIdx.z * sB + (long long)bn * BN;
  C += (long long)blockIdx.z * sC;
  const int k_begin = tri ? max(bm * BM, bn * BN) : 0;
  const int ktiles = (K - k_begin) / BK;

  auto load_stage = [&](int stage, int kt) {
    const int k0 = k_begin + kt * BK;
    double* as = As + stage * A_STAGE;
    double* bs = Bs + stage * B_STAGE;
#pragma unroll
    for (int i = 0; i < 4; ++i) {  // A: 128 rows x 8 chunks of 2 doubles
      const int c = tid + i * THREADS, r = c >> 3, kc = (c & 7) * 2;
      cp_async16(as + r * LDA_S + kc, A + (long long)r * lda + k0 + kc);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {  // B: 16 rows x 64 chunks of 2 doubles
      const int c = tid + i * THREADS, r = c >> 6, nc = (c & 63) * 2;
      cp_async16(bs + r * LDB_S + nc, B + (long long)(k0 + r) * ldb + nc);
    }
  };

  double acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < ktiles) load_stage(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < ktiles; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();  // stage kt landed for every thread; stage kt - 1 is no longer read
    if (kt + STAGES - 1 < ktiles) load_stage((kt + STAGES - 1) % STAGES, kt + STAGES - 1);
    cp_async_commit();
    const double* as = As + (kt % STAGES) * A_STAGE + (wm + g) * LDA_S + t;
    const double* bs = Bs + (kt % STAGES) * B_STAGE + t * LDB_S + wn + g;
    double b[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) b[j][i] = bs[i * 4 * LDB_S + j * 8];
#pragma unroll
    for (int mi = 0; mi < 4; ++mi) {
      double a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = as[(mi * 16 + 8 * (i & 1)) * LDA_S + 4 * (i >> 1)];
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma16816(acc[mi][j], a, b[j]);
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int mi = 0; mi < 4; ++mi)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long row = (long long)bm * BM + wm + mi * 16 + g + 8 * h;
        const int col = bn * BN + wn + j * 8 + 2 * t;
        const double v0 = alpha * acc[mi][j][2 * h], v1 = alpha * acc[mi][j][2 * h + 1];
        if (col_map) {
          C[row * ldc + col_map[col]] = v0;
          C[row * ldc + col_map[col + 1]] = v1;
        } else {
          double2* p = reinterpret_cast<double2*>(C + row * ldc + col);
          if (beta == 0.0) {
            *p = make_double2(v0, v1);
          } else {
            const double2 c = *p;
            *p = make_double2(v0 + beta * c.x, v1 + beta * c.y);
          }
        }
      }
}

// Host launcher (stream-ordered, no synchronisation).  Returns the launch error, if any.
inline cudaError_t dgemm(cudaStream_t st, int M, int N, int K, double alpha, const double* A, int lda, long long sA, const double* B,
                         int ldb, long long sB, double beta, double* C, int ldc, long long sC, int batch, bool tri = false,
                         const int* col_map = nullptr) {
  if (M <= 0 || N <= 0 || batch <= 0) return cudaSuccess;
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(dgemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  dgemm_kernel<<<dim3(N / BN, M / BM, batch), THREADS, SMEM_BYTES, st>>>(K, tri ? 1 : 0, alpha, A, lda, sA, B, ldb, sB, beta, C, ldc,
                                                                         sC, col_map);
  return cudaGetLastError();
}

}  // namespace dtc
}  // namespace b200
