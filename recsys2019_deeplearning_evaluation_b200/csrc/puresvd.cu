// K9: PureSVD, scikit-learn's randomized_svd(URM, n_components=k, random_state=seed) as the reference's PureSVDRecommender
// runs it (sklearn/utils/extmath.py: _randomized_svd, _randomized_range_finder).
//
// A is the URM (n_users >= n_items) or URM^T (transpose), so that A [ma, d] has d = min(n_users, n_items) columns.  The
// range finder works on r = min(n_random, d) columns, the first r of the host's draw Omega [d, n_random]:
//   n_iter times:  Y = A Q, Q = orth(Y);  Z = A^T Q, Q = orth(Z)        (scikit-learn: LU, the same spans)
//   Q = orth(A Q) (two passes);  B^T = A^T Q;  B B^T = (B^T)^T B^T = W diag(lambda) W^T;  s = sqrt(lambda) descending
//   Q side = Q W,  other side (V S) = B^T W;  the user side carries svd_flip's sign decision.
// Tall matrices are fp32 (as scikit-learn's float32 run keeps them), every product accumulates in fp64, the r x r matrices
// are fp64.  Kernels:
//   transpose    CSR -> CSR of the transpose: stable radix sort of the column ids, so every output row stays sorted
//   spmm, gram   K8's (spmm_gram.cuh)
//   tall_small   out [m, c] = in [m, r] (fp32) x C [r, c] (fp64), 64 rows per block staged in shared memory (in place
//                when c == r), C streamed in 32 x 32 tiles
//   jacobi       one round of the parallel cyclic Jacobi method on an r x r symmetric fp64 matrix: the circle method
//                pairs every index once per round, all r/2 rotations are applied together (A <- J^T A J, V <- V J)
//   orth         SVQB: G = Y^T Y, D = diag(G)^-1/2, D G D = W diag(lambda) W^T, Y <- Y D W diag(lambda)^-1/2; eigenvalues
//                at or below n_random * eps64 * lambda_max give zero columns
//   flip         per component, the user-side entry of largest |.| (lowest row on ties) is made positive on both sides
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <float.h>

#include <algorithm>
#include <cmath>

#include "spmm_gram.cuh"

namespace b200 {
namespace svd {

using nmf::F_MAX;
using nmf::WARPS;
constexpr int R_MAX = F_MAX;  // columns of the sketch
constexpr int TR = 64;        // rows per block of tall_small_kernel
constexpr int MAX_SWEEPS = 60;
constexpr int JACOBI_ELEMS = 1024;  // matrix elements per block of jacobi_round_kernel

// ---- CSR transpose ------------------------------------------------------------------------------------------------
// rowid[q] = the row whose range [ptr[row], ptr[row + 1]) holds q
__global__ void row_of_kernel(long long nnz, int n_rows, const int* __restrict__ ptr, int* __restrict__ rowid, int* __restrict__ iota) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_rows - 1;  // the last row with ptr[row] <= q
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (ptr[mid] <= q) lo = mid;
      else hi = mid - 1;
    }
    rowid[q] = lo;
    iota[q] = (int)q;
  }
}

__global__ void count_cols_kernel(long long nnz, const int* __restrict__ idx, int* __restrict__ cnt) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x)
    atomicAdd(cnt + idx[q], 1);
}

__global__ void gather_transpose_kernel(long long nnz, const int* __restrict__ perm, const int* __restrict__ rowid,
                                        const float* __restrict__ val, int* __restrict__ out_idx, float* __restrict__ out_val) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x) {
    const int p = perm[q];
    out_idx[q] = rowid[p];
    out_val[q] = val[p];
  }
}

void csr_transpose(cudaStream_t st, int n_rows, int n_cols, long long nnz, const int* ptr, const int* idx, const float* val,
                   int* out_ptr, int* out_idx, float* out_val) {
  DevBuf<int> cnt((size_t)n_cols + 1);
  B200_CUDA(cudaMemsetAsync(cnt.get(), 0, sizeof(int) * ((size_t)n_cols + 1), st));
  const unsigned grid = (unsigned)std::min<long long>(4096, std::max<long long>(1, div_up(nnz, 256)));
  size_t tb_scan = 0, tb_sort = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb_scan, cnt.get(), out_ptr, n_cols + 1, st));
  if (nnz > 0) {
    int end_bit = 1;
    while ((1ll << end_bit) < (long long)n_cols) ++end_bit;
    DevBuf<int> rowid(nnz), iota(nnz), keys(nnz), perm(nnz);
    B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, idx, keys.get(), iota.get(), perm.get(), (int)nnz, 0, end_bit, st));
    DevBuf<unsigned char> tmp(std::max(tb_scan, tb_sort) + 16);
    count_cols_kernel<<<grid, 256, 0, st>>>(nnz, idx, cnt.get());
    row_of_kernel<<<grid, 256, 0, st>>>(nnz, n_rows, ptr, rowid.get(), iota.get());
    B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tb_sort, idx, keys.get(), iota.get(), perm.get(), (int)nnz, 0, end_bit, st));
    gather_transpose_kernel<<<grid, 256, 0, st>>>(nnz, perm.get(), rowid.get(), val, out_idx, out_val);
    B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb_scan, cnt.get(), out_ptr, n_cols + 1, st));
    B200_CUDA(cudaGetLastError());
    count_launch(7);
    B200_CUDA(cudaStreamSynchronize(st));  // the temporaries are freed on return
  } else {
    DevBuf<unsigned char> tmp(tb_scan + 16);
    B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb_scan, cnt.get(), out_ptr, n_cols + 1, st));
    count_launch(1);
    B200_CUDA(cudaStreamSynchronize(st));
  }
}

// ---- tall x small -------------------------------------------------------------------------------------------------
// out[i, :c] = in[i, :r] C  (C [r, c] row-major fp64), accumulated in fp64 and rounded once.  The block reads all its rows
// into shared memory before it writes any, so out may be in when c == r.
__global__ void __launch_bounds__(256) tall_small_kernel(int n, int r, int c, const float* in, const double* __restrict__ C,
                                                         float* out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* Cs = reinterpret_cast<double*>(smem);              // [32][32]
  float* Is = reinterpret_cast<float*>(smem + 32 * 32 * 8);  // [TR][r]
  const int ty = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * TR;
  for (int e = threadIdx.x; e < TR * r; e += blockDim.x) {
    const int rr = e / r, cc = e - rr * r;
    Is[e] = r0 + rr < n ? in[(size_t)(r0 + rr) * r + cc] : 0.f;
  }
  __syncthreads();
  for (int c0 = 0; c0 < c; c0 += 32) {
    double acc[TR / WARPS];
#pragma unroll
    for (int j = 0; j < TR / WARPS; ++j) acc[j] = 0.0;
    for (int k0 = 0; k0 < r; k0 += 32) {
      for (int e = threadIdx.x; e < 1024; e += blockDim.x) {
        const int kk = e >> 5, cc = e & 31;
        Cs[e] = k0 + kk < r && c0 + cc < c ? C[(size_t)(k0 + kk) * c + c0 + cc] : 0.0;
      }
      __syncthreads();
      const int kn = min(32, r - k0);
      for (int kk = 0; kk < kn; ++kk) {
        const double g = Cs[kk * 32 + lane];
#pragma unroll
        for (int j = 0; j < TR / WARPS; ++j) acc[j] += (double)Is[(ty + WARPS * j) * r + k0 + kk] * g;
      }
      __syncthreads();
    }
    const int cc = c0 + lane;
    if (cc < c) {
#pragma unroll
      for (int j = 0; j < TR / WARPS; ++j) {
        const int rr = ty + WARPS * j;
        if (r0 + rr < n) out[(size_t)(r0 + rr) * c + cc] = (float)acc[j];
      }
    }
  }
}

// ---- parallel cyclic Jacobi -----------------------------------------------------------------------------------------
// Round t (0 <= t < n - 1) of the circle method on n (even) indices: n - 1 meets t, every other i meets (2t - i) mod (n - 1).
// Indices >= r (the one pad index when r is odd) take no rotation.
__device__ __forceinline__ int partner(int i, int t, int n) {
  if (i == n - 1) return t;
  if (i == t) return n - 1;
  const int p = (2 * t - i) % (n - 1);
  return p < 0 ? p + n - 1 : p;
}

// A' = J^T A J and V' = V J for all rotations of round t.  Index i of pair (p, q), p < q, has J[:, i] = c e_i + g e_partner,
// g = -s for p and +s for q (Golub & Van Loan's sym.schur2 zeroes A'[p, q], which is then stored as an exact zero).  Every
// element of A' is computed from the upper triangle, so A stays exactly symmetric.
__global__ void __launch_bounds__(256) jacobi_round_kernel(int r, int n, int t, const double* __restrict__ A, double* __restrict__ A2,
                                                           const double* __restrict__ V, double* __restrict__ V2) {
  __shared__ double cs[R_MAX], gs[R_MAX];
  __shared__ int ps[R_MAX];
  for (int i = threadIdx.x; i < r; i += blockDim.x) {
    const int pi = partner(i, t, n);
    double c = 1.0, g = 0.0;
    if (pi < r) {
      const int p = min(i, pi), q = max(i, pi);
      const double apq = A[(size_t)p * r + q];
      if (apq != 0.0) {
        const double tau = (A[(size_t)q * r + q] - A[(size_t)p * r + p]) / (2.0 * apq);
        const double tt = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
        c = 1.0 / sqrt(1.0 + tt * tt);
        const double s = tt * c;
        g = i == p ? -s : s;
      }
    }
    cs[i] = c;
    gs[i] = g;
    ps[i] = pi < r ? pi : i;
  }
  __syncthreads();
  const long long rr = (long long)r * r;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < 2 * rr; e += (long long)gridDim.x * blockDim.x) {
    if (e < rr) {
      const int i = (int)(e / r), j = (int)(e % r);
      const int a = min(i, j), b = max(i, j), pa = ps[a], pb = ps[b];
      double v;
      if (pa == b && gs[a] != 0.0) {
        v = 0.0;
      } else {
        const double ca = cs[a], ga = gs[a], cb = cs[b], gb = gs[b];
        // A[x][y] for x <= y read from the upper triangle
        auto at = [&](int x, int y) { return x <= y ? A[(size_t)x * r + y] : A[(size_t)y * r + x]; };
        v = ca * cb * at(a, b);
        if (gb != 0.0) v += ca * gb * at(a, pb);
        if (ga != 0.0) v += ga * cb * at(pa, b);
        if (ga != 0.0 && gb != 0.0) v += ga * gb * at(pa, pb);
      }
      A2[e] = v;
    } else {
      const long long f = e - rr;
      const int k = (int)(f / r), j = (int)(f % r);
      double v = cs[j] * V[f];
      if (gs[j] != 0.0) v += gs[j] * V[(size_t)k * r + ps[j]];
      V2[f] = v;
    }
  }
}

// out[0] = sum of the squared off-diagonal entries, out[1] = sum of all squared entries (one block, fixed order)
__global__ void __launch_bounds__(1024) offnorm_kernel(int r, const double* __restrict__ A, double* __restrict__ out) {
  __shared__ double so[1024], st[1024];
  double off = 0.0, tot = 0.0;
  for (long long e = threadIdx.x; e < (long long)r * r; e += blockDim.x) {
    const double a = A[e], a2 = a * a;
    tot += a2;
    if (e / r != e % r) off += a2;
  }
  so[threadIdx.x] = off;
  st[threadIdx.x] = tot;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      so[threadIdx.x] += so[threadIdx.x + w];
      st[threadIdx.x] += st[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = so[0];
    out[1] = st[0];
  }
}

// order[k] = the index of the k-th largest diagonal entry of A (lower index first on ties); lam[k] = that entry
__global__ void __launch_bounds__(1024) sort_desc_kernel(int r, const double* __restrict__ A, int* __restrict__ order,
                                                         double* __restrict__ lam) {
  for (int i = threadIdx.x; i < r; i += blockDim.x) {
    const double li = A[(size_t)i * r + i];
    int rank = 0;
    for (int j = 0; j < r; ++j) {
      const double lj = A[(size_t)j * r + j];
      rank += lj > li || (lj == li && j < i);
    }
    order[rank] = i;
    lam[rank] = li;
  }
}

__global__ void identity_kernel(int r, double* __restrict__ M) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e < (long long)r * r) M[e] = e / r == e % r ? 1.0 : 0.0;
}

// ---- SVQB -----------------------------------------------------------------------------------------------------------
// A = D G D with D = diag(G)^-1/2 (0 where G[i, i] = 0), V = I; d[i] = D[i, i]
__global__ void svqb_scale_kernel(int r, const double* __restrict__ G, double* __restrict__ A, double* __restrict__ V,
                                  double* __restrict__ d) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)r * r) return;
  const int i = (int)(e / r), j = (int)(e % r);
  const double gi = G[(size_t)i * r + i], gj = G[(size_t)j * r + j];
  const double di = gi > 0.0 ? 1.0 / sqrt(gi) : 0.0, dj = gj > 0.0 ? 1.0 / sqrt(gj) : 0.0;
  A[e] = G[e] * di * dj;
  V[e] = i == j ? 1.0 : 0.0;
  if (j == 0) d[i] = di;
}

// C = D W diag(lambda)^-1/2, columns with lambda_j <= n_random * eps64 * lambda_max set to zero
__global__ void svqb_coef_kernel(int r, int n_random, const double* __restrict__ A, const double* __restrict__ W,
                                 const double* __restrict__ d, double* __restrict__ C) {
  __shared__ double lmax;
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int i = 0; i < r; ++i) m = fmax(m, A[(size_t)i * r + i]);
    lmax = m;
  }
  __syncthreads();
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)r * r) return;
  const int i = (int)(e / r), j = (int)(e % r);
  const double lj = A[(size_t)j * r + j];
  C[e] = lj > n_random * DBL_EPSILON * lmax ? d[i] * W[e] / sqrt(lj) : 0.0;
}

// ---- step 6 ---------------------------------------------------------------------------------------------------------
// Cq[:, j] = W[:, order[j]] * sq_j and Cb[:, j] = W[:, order[j]] * sb_j for j < kp, with s_j = sqrt(max(lambda_j, 0)):
// no transpose (Q side = users):  sq = 1, sb = 1;  transpose (Q side = items):  sq = s_j, sb = 1 / s_j, or 0 when
// s_j <= n_random * eps64 * s_1.  s_out[j] = s_j.
__global__ void final_coef_kernel(int r, int kp, int n_random, int transpose, const double* __restrict__ W, const int* __restrict__ order,
                                  const double* __restrict__ lam, double* __restrict__ Cq, double* __restrict__ Cb,
                                  double* __restrict__ s_out) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (long long)r * kp) return;
  const int i = (int)(e / kp), j = (int)(e % kp);
  const double s1 = sqrt(fmax(lam[0], 0.0)), sj = sqrt(fmax(lam[j], 0.0));
  const double w = W[(size_t)i * r + order[j]];
  if (!transpose) {
    Cq[e] = w;
    Cb[e] = w;
  } else {
    Cq[e] = w * sj;
    Cb[e] = sj > n_random * DBL_EPSILON * s1 ? w / sj : 0.0;
  }
  if (i == 0) s_out[j] = sj;
}

// sign[j] = -1 when the entry of largest |.| in column j of U [n, k] (lowest row on ties) is negative, else +1
__global__ void __launch_bounds__(1024) flip_sign_kernel(int n, int k, const float* __restrict__ U, float* __restrict__ sign) {
  __shared__ float bv[1024];
  __shared__ int bi[1024];
  const int j = blockIdx.x;
  float best = -1.f;
  int at = n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float a = fabsf(U[(size_t)i * k + j]);
    if (a > best) { best = a; at = i; }  // rows visited in increasing order: the first maximum stays
  }
  bv[threadIdx.x] = best;
  bi[threadIdx.x] = at;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      const float ob = bv[threadIdx.x + w];
      const int oi = bi[threadIdx.x + w];
      if (ob > bv[threadIdx.x] || (ob == bv[threadIdx.x] && oi < bi[threadIdx.x])) {
        bv[threadIdx.x] = ob;
        bi[threadIdx.x] = oi;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) sign[j] = bi[0] < n && U[(size_t)bi[0] * k + j] < 0.f ? -1.f : 1.f;
}

// M[i, j] *= sign[j] for M [n, k]
__global__ void scale_cols_kernel(long long n, int k, const float* __restrict__ sign, float* __restrict__ M) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n * k; e += (long long)gridDim.x * blockDim.x)
    M[e] *= sign[e % k];
}

struct Csr {
  int n_rows;
  const int* ptr;
  const int* idx;
  const float* val;
};

// Workspace and launches for r-column tall operands of n_a or n_b rows.
struct Svd {
  cudaStream_t st;
  int r, n_random;
  DevBuf<double> split_part, G, A0, A1, V0, V1, d, C, lam, offs;
  DevBuf<int> order;

  Svd(cudaStream_t s, int r_, int n_random_, int n_a, int n_b) : st(s), r(r_), n_random(n_random_) {
    const int tiles = (r + 31) / 32;
    // the split count is not monotonic in the row count: size for both
    const size_t splits = std::max(nmf::n_splits(n_a, tiles * tiles), nmf::n_splits(n_b, tiles * tiles));
    split_part.alloc(splits * r * r);
    for (DevBuf<double>* b : {&G, &A0, &A1, &V0, &V1, &C}) b->alloc((size_t)r * r);
    d.alloc(r);
    lam.alloc(r);
    offs.alloc(2);
    order.alloc(r);
    const int bytes = 32 * 32 * (int)sizeof(double) + TR * R_MAX * (int)sizeof(float);
    B200_CUDA(cudaFuncSetAttribute(tall_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  }

  void spmm(const Csr& A, const float* M, float* out) {
    nmf::spmm_kernel<<<div_up(A.n_rows, WARPS), 256, 0, st>>>(A.n_rows, A.ptr, A.idx, A.val, M, r, out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  // G = M^T M (fp64) over the n rows of M [n, r]
  void gram(const float* M, int n, double* out) {
    const int tiles = (r + 31) / 32;
    const int per = nmf::split_rows(n, tiles * tiles);
    const int splits = (int)div_up(n, per);
    B200_REQUIRE((size_t)splits * r * r <= split_part.n, "b200_puresvd: Gram split workspace too small (%d splits)", splits);
    nmf::gram_partial_kernel<<<dim3(tiles * tiles, splits), 256, 0, st>>>(n, r, M, per, split_part.get());
    nmf::sum_splits_kernel<<<div_up((long long)r * r, 256), 256, 0, st>>>(split_part.get(), splits, (long long)r * r, out);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  }
  // out [n, c] = in [n, r] C [r, c]
  void tall_small(const float* in, int n, const double* Cm, int c, float* out) {
    if (n == 0) return;
    const size_t bytes = 32 * 32 * sizeof(double) + (size_t)TR * r * sizeof(float);
    tall_small_kernel<<<div_up(n, TR), 256, bytes, st>>>(n, r, c, in, Cm, out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  // Eigendecomposition of the symmetric matrix in A0: on return the eigenvalues are the diagonal of A0, the eigenvectors the
  // columns of V0 (unsorted).  V0 must hold the start basis (the identity).  Sweeps run until the off-diagonal part is
  // below 1e-17 of the Frobenius norm; the host reads two doubles per sweep.
  void jacobi() {
    const int n = r + (r & 1);
    const unsigned blocks = div_up(2ll * r * r, JACOBI_ELEMS);
    for (int sweep = 0; sweep <= MAX_SWEEPS; ++sweep) {
      offnorm_kernel<<<1, 1024, 0, st>>>(r, A0.get(), offs.get());
      B200_CUDA(cudaGetLastError());
      count_launch();
      double h[2];
      B200_CUDA(cudaMemcpyAsync(h, offs.get(), sizeof(h), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      if (!(h[0] > 1e-34 * h[1])) return;
      B200_REQUIRE(sweep < MAX_SWEEPS, "b200_puresvd: the Jacobi eigensolver did not converge in %d sweeps (r = %d)", MAX_SWEEPS, r);
      for (int t = 0; t < n - 1; ++t) {
        jacobi_round_kernel<<<blocks, 256, 0, st>>>(r, n, t, A0.get(), A1.get(), V0.get(), V1.get());
        std::swap(A0, A1);
        std::swap(V0, V1);
      }
      B200_CUDA(cudaGetLastError());
      count_launch(n - 1);
    }
  }
  void sort_desc() {
    sort_desc_kernel<<<1, 1024, 0, st>>>(r, A0.get(), order.get(), lam.get());
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  // eigendecomposition of the symmetric r x r matrix S (which may be A0 itself)
  void eigh(const double* S) {
    if (S != A0.get()) B200_CUDA(cudaMemcpyAsync(A0.get(), S, sizeof(double) * r * r, cudaMemcpyDeviceToDevice, st));
    identity(V0.get());
    jacobi();
  }
  void identity(double* M) {
    identity_kernel<<<div_up((long long)r * r, 256), 256, 0, st>>>(r, M);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  // Y [n, r] <- an orthonormal basis of its span (SVQB, `passes` times); dropped directions are zero columns
  void orth(float* Y, int n, int passes) {
    for (int p = 0; p < passes; ++p) {
      gram(Y, n, G.get());
      svqb_scale_kernel<<<div_up((long long)r * r, 256), 256, 0, st>>>(r, G.get(), A0.get(), V0.get(), d.get());
      B200_CUDA(cudaGetLastError());
      count_launch();
      jacobi();
      svqb_coef_kernel<<<div_up((long long)r * r, 256), 256, 0, st>>>(r, n_random, A0.get(), V0.get(), d.get(), C.get());
      B200_CUDA(cudaGetLastError());
      count_launch();
      tall_small(Y, n, C.get(), r, Y);
    }
  }
};

// svd_flip on the user side U [n_u, k]; the other side O [n_o, k] takes the same signs
void flip(cudaStream_t st, float* U, int n_u, float* O, int n_o, int k) {
  DevBuf<float> sign(k);
  flip_sign_kernel<<<k, 1024, 0, st>>>(n_u, k, U, sign.get());
  const unsigned gu = std::min<unsigned>(4096, std::max(1u, div_up((long long)n_u * k, 256)));
  const unsigned go = std::min<unsigned>(4096, std::max(1u, div_up((long long)n_o * k, 256)));
  scale_cols_kernel<<<gu, 256, 0, st>>>(n_u, k, sign.get(), U);
  scale_cols_kernel<<<go, 256, 0, st>>>(n_o, k, sign.get(), O);
  B200_CUDA(cudaGetLastError());
  count_launch(3);
  B200_CUDA(cudaStreamSynchronize(st));  // sign is freed on return
}

}  // namespace svd
}  // namespace b200

using namespace b200;
using namespace b200::svd;

extern "C" {

int b200_csr_transpose_device(int n_rows, int n_cols, int64_t nnz, const int32_t* d_ptr, const int32_t* d_idx, const float* d_val,
                              int32_t* d_out_ptr, int32_t* d_out_idx, float* d_out_val, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n_rows >= 1 && n_cols >= 1 && nnz >= 0 && nnz < (1ll << 31), "b200_csr_transpose: bad shape (%d x %d, nnz %lld)",
                 n_rows, n_cols, (long long)nnz);
    B200_REQUIRE(d_ptr && d_out_ptr && (nnz == 0 || (d_idx && d_val && d_out_idx && d_out_val)), "b200_csr_transpose: NULL argument");
    csr_transpose((cudaStream_t)stream, n_rows, n_cols, nnz, d_ptr, d_idx, d_val, d_out_ptr, d_out_idx, d_out_val);
  });
}

int b200_puresvd_device(int n_users, int n_items, const int32_t* d_x_ptr, const int32_t* d_x_idx, const float* d_x_val,
                        const int32_t* d_xt_ptr, const int32_t* d_xt_idx, const float* d_xt_val, const float* d_omega, int n_random,
                        int k, int n_iter, int transpose, float* d_user, float* d_item, double* d_s, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n_users >= 1 && n_items >= 1, "b200_puresvd: bad shape (%d x %d)", n_users, n_items);
    B200_REQUIRE(k >= 1 && n_random > k && n_random <= R_MAX, "b200_puresvd: need 1 <= k < n_random <= %d (k %d, n_random %d)", R_MAX,
                 k, n_random);
    B200_REQUIRE(n_iter >= 0, "b200_puresvd: bad n_iter %d", n_iter);
    B200_REQUIRE((transpose != 0) == (n_users < n_items), "b200_puresvd: transpose must be n_users < n_items");
    // the column ids and values may be NULL when the URM has no entries
    B200_REQUIRE(d_x_ptr && d_xt_ptr && d_omega && d_user && d_item && d_s, "b200_puresvd: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const Csr X{n_users, d_x_ptr, d_x_idx, d_x_val}, Xt{n_items, d_xt_ptr, d_xt_idx, d_xt_val};
    const Csr& A = transpose ? Xt : X;   // [ma, d]
    const Csr& At = transpose ? X : Xt;  // [d, ma]
    const int ma = A.n_rows, d = At.n_rows;
    const int r = std::min(n_random, d), kp = std::min(k, d);
    Svd s(st, r, n_random, ma, d);
    DevBuf<float> Q((size_t)d * r), Y((size_t)ma * r);
    DevBuf<double> Cq((size_t)r * kp), Cb((size_t)r * kp);
    B200_CUDA(cudaMemcpy2DAsync(Q.get(), sizeof(float) * r, d_omega, sizeof(float) * n_random, sizeof(float) * r, d,
                                cudaMemcpyDeviceToDevice, st));
    for (int it = 0; it < n_iter; ++it) {
      s.spmm(A, Q.get(), Y.get());
      s.orth(Y.get(), ma, 1);
      s.spmm(At, Y.get(), Q.get());
      s.orth(Q.get(), d, 1);
    }
    s.spmm(A, Q.get(), Y.get());
    s.orth(Y.get(), ma, 2);  // Y = Q of scikit-learn
    s.spmm(At, Y.get(), Q.get());  // Q = B^T
    s.gram(Q.get(), d, s.G.get());  // B B^T
    s.eigh(s.G.get());
    s.sort_desc();
    final_coef_kernel<<<div_up((long long)r * kp, 256), 256, 0, st>>>(r, kp, n_random, transpose, s.V0.get(), s.order.get(),
                                                                       s.lam.get(), Cq.get(), Cb.get(), d_s);
    B200_CUDA(cudaGetLastError());
    count_launch();
    float* q_side = transpose ? d_item : d_user;
    float* b_side = transpose ? d_user : d_item;
    s.tall_small(Y.get(), ma, Cq.get(), kp, q_side);
    s.tall_small(Q.get(), d, Cb.get(), kp, b_side);
    flip(st, d_user, n_users, d_item, n_items, kp);
  });
}

int b200_svd_debug_device(int op, int n_rows, int n_cols, int arg, void* d_a, void* d_b, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n_rows >= 1 && n_cols >= 1 && n_cols <= R_MAX && d_a, "b200_svd_debug: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (op == 0) {
      B200_REQUIRE(arg >= 1, "b200_svd_debug: bad pass count %d", arg);
      Svd s(st, n_cols, n_cols, n_rows, n_rows);
      s.orth((float*)d_a, n_rows, arg);
    } else if (op == 1) {
      B200_REQUIRE(n_rows == n_cols && d_b, "b200_svd_debug: the eigensolver takes a square matrix and an output");
      const int r = n_cols;
      Svd s(st, r, r, r, r);
      s.eigh((const double*)d_a);
      s.sort_desc();
      double* out = (double*)d_b;
      B200_CUDA(cudaMemcpyAsync(out, s.lam.get(), sizeof(double) * r, cudaMemcpyDeviceToDevice, st));
      // eigenvector columns in the sorted order: out[r + i * r + j] = V[i, order[j]]
      final_coef_kernel<<<div_up((long long)r * r, 256), 256, 0, st>>>(r, r, r, 0, s.V0.get(), s.order.get(), s.lam.get(),
                                                                        out + r, s.C.get(), s.d.get());
      B200_CUDA(cudaGetLastError());
      count_launch();
    } else if (op == 2) {
      B200_REQUIRE(arg >= 0 && (arg == 0 || d_b), "b200_svd_debug: bad other side");
      flip(st, (float*)d_a, n_rows, (float*)d_b, arg, n_cols);
    } else {
      B200_REQUIRE(false, "b200_svd_debug: bad op %d", op);
    }
    B200_CUDA(cudaStreamSynchronize(st));
  });
}

}  // extern "C"
