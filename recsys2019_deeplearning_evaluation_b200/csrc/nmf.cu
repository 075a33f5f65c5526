// K8: non-negative matrix factorisation, scikit-learn's NMF(init="random", alpha_W=0) as the reference's NMFRecommender runs it
// (sklearn/decomposition/_nmf.py: _fit_multiplicative_update, _fit_coordinate_descent, _cdnmf_fast.pyx).
//
// State: W [n_users, f] and Ht = H^T [n_items, f], row-major fp32.  X is the URM as CSR, X^T its CSR transpose (the CSC).
// Every product accumulates in fp64 and is rounded once to fp32 (factors, X H^T) or kept in fp64 (Grams, column sums,
// losses).  Kernels:
//   spmm         out[r] = sum over (j, x) in row r of a CSR:  x * M[j]              one warp per row, f <= F_MAX
//   gram         G = M^T M (fp64), 32 x 32 output tiles, rows split over the grid, partials summed in a fixed order
//   colsum       s = column sums of M (fp64), the same split
//   mu_fro       A[i] *= num[i] / (A[i] G)  (zero denominator -> EPS), A[i] staged in shared memory so that the block can
//                overwrite its rows while it streams G in 32 x 32 tiles
//   kl           fused SDDMM + SpMM: per row r of a CSR, A[r] *= (sum over (j, x) of x / max(A[r] . B[j], EPS) * B[j]) / s
//   cd_sweep     one coordinate-descent pass over the components, one warp per row with the row in shared memory
// The host loop of b200_nmf_solve_device reads one double per stopping test and nothing else.
#include <float.h>

#include <algorithm>
#include <cmath>

#include "spmm_gram.cuh"

namespace b200 {
namespace nmf {

constexpr int TR = 64;  // rows per block of mu_fro_update_kernel
constexpr double EPS = 1.1920928955078125e-07;  // np.finfo(np.float32).eps, _nmf.py EPSILON
constexpr int DOT_BLOCKS = 1024;

// P[split][c] = sum over the split's rows of M[i, c]; blockIdx.x = 32-column tile, blockIdx.y = split
__global__ void __launch_bounds__(256) colsum_partial_kernel(int n, int f, const float* __restrict__ M, int rows_per_split,
                                                             double* __restrict__ P) {
  __shared__ double part[WARPS][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * 32 + lane;
  const int r_begin = blockIdx.y * rows_per_split, r_end = min(n, r_begin + rows_per_split);
  double acc = 0.0;
  if (c < f)
    for (int r = r_begin + warp; r < r_end; r += WARPS) acc += (double)M[(size_t)r * f + c];
  part[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && c < f) {
    double s = 0.0;
    for (int w = 0; w < WARPS; ++w) s += part[w][lane];
    P[(size_t)blockIdx.y * f + c] = s;
  }
}

// A[i, c] = A[i, c] * (num[i, c] / den) with den = (A[i, :] G)[c], 0 -> EPS  (_multiplicative_update_w / _h, Frobenius)
__global__ void __launch_bounds__(256) mu_fro_update_kernel(int n, int f, float* __restrict__ A, const float* __restrict__ num,
                                                            const double* __restrict__ G) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* Gs = reinterpret_cast<double*>(smem);           // [32][32]
  float* As = reinterpret_cast<float*>(smem + 32 * 32 * 8);  // [TR][f]
  const int ty = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * TR;
  for (int e = threadIdx.x; e < TR * f; e += blockDim.x) {
    const int rr = e / f, cc = e - rr * f;
    As[e] = r0 + rr < n ? A[(size_t)(r0 + rr) * f + cc] : 0.f;
  }
  __syncthreads();
  for (int c0 = 0; c0 < f; c0 += 32) {
    double acc[TR / WARPS];
#pragma unroll
    for (int j = 0; j < TR / WARPS; ++j) acc[j] = 0.0;
    for (int k0 = 0; k0 < f; k0 += 32) {
      for (int e = threadIdx.x; e < 1024; e += blockDim.x) {
        const int kk = e >> 5, cc = e & 31;
        Gs[e] = k0 + kk < f && c0 + cc < f ? G[(size_t)(k0 + kk) * f + c0 + cc] : 0.0;
      }
      __syncthreads();
      const int kn = min(32, f - k0);
      for (int kk = 0; kk < kn; ++kk) {
        const double g = Gs[kk * 32 + lane];
#pragma unroll
        for (int j = 0; j < TR / WARPS; ++j) acc[j] += (double)As[(ty + WARPS * j) * f + k0 + kk] * g;
      }
      __syncthreads();
    }
    const int c = c0 + lane;
    if (c < f) {
#pragma unroll
      for (int j = 0; j < TR / WARPS; ++j) {
        const int rr = ty + WARPS * j;
        if (r0 + rr < n) {
          const double den = acc[j] == 0.0 ? EPS : acc[j];
          const size_t o = (size_t)(r0 + rr) * f + c;
          A[o] = (float)((double)As[rr * f + c] * ((double)num[o] / den));
        }
      }
    }
  }
}

// Kullback-Leibler multiplicative update of the rows of A against B over the CSR (ptr, idx, val) (row r of A <-> row r of the
// CSR, column j <-> row j of B):  wh = A[r] . B[j] at the non-zeros, clamped below at EPS;  A[r] *= (sum x / wh * B[j]) / s,
// s = d_sum (a column sum of the other factor) with 0 -> 1 when zero_to_one (W_sum in _multiplicative_update_h), then
// 0 -> EPS.  zero_small: A[r, c] < float64 eps -> 0 (_fit_multiplicative_update, beta_loss <= 1, after the H step).
// With d_sum NULL the kernel instead writes, per row, sum over the non-zeros with x > EPS of x log(x / wh) - x to row_loss.
__global__ void __launch_bounds__(256) kl_kernel(int n_rows, const int* __restrict__ ptr, const int* __restrict__ idx,
                                                 const float* __restrict__ val, float* __restrict__ A, const float* __restrict__ B,
                                                 int f, const double* __restrict__ d_sum, int zero_to_one, int zero_small,
                                                 double* __restrict__ row_loss) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  float a[KMAX];
  double acc[KMAX];
  float* ar = A + (size_t)row * f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    const int c = lane + 32 * k;
    a[k] = c < f ? ar[c] : 0.f;
    acc[k] = 0.0;
  }
  double loss = 0.0;
  const int s = ptr[row], e = ptr[row + 1];
  for (int q0 = s; q0 < e; q0 += 32) {
    int jj = 0;
    float xx = 0.f;
    if (q0 + lane < e) { jj = idx[q0 + lane]; xx = val[q0 + lane]; }
    const int cnt = min(32, e - q0);
    for (int t = 0; t < cnt; ++t) {
      const int j = __shfl_sync(0xffffffffu, jj, t);
      const double x = __shfl_sync(0xffffffffu, xx, t);
      const float* br = B + (size_t)j * f;
      float b[KMAX];
      double d = 0.0;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const int c = lane + 32 * k;
        b[k] = c < f ? br[c] : 0.f;
        d += (double)a[k] * (double)b[k];
      }
      d = warp_sum(d);
      const double wh = d < EPS ? EPS : d;
      if (d_sum) {
        const double r = x / wh;
#pragma unroll
        for (int k = 0; k < KMAX; ++k) acc[k] += r * (double)b[k];
      } else if (x > EPS) {
        loss += x * log(x / wh) - x;
      }
    }
  }
  if (!d_sum) {
    if (lane == 0) row_loss[row] = loss;
    return;
  }
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    const int c = lane + 32 * k;
    if (c < f) {
      double den = d_sum[c];
      if (zero_to_one && den == 0.0) den = 1.0;
      if (den == 0.0) den = EPS;
      double v = (double)a[k] * (acc[k] / den);
      if (zero_small && v < DBL_EPSILON) v = 0.0;
      ar[c] = (float)v;
    }
  }
}

// _update_cdnmf_fast for one row per warp: for t = 0 .. f-1 in order, grad = (A[i] . HHt[t]) - XHt[i, t], the projected
// gradient's |.| goes to the violation, and A[i, t] = max(A[i, t] - grad / HHt[t, t], 0) unless HHt[t, t] == 0.  The row is
// kept in fp64 in shared memory during the pass.  viol_partial[block] = the block's violation.
__global__ void __launch_bounds__(256) cd_sweep_kernel(int n_rows, int f, float* __restrict__ A, const double* __restrict__ HHt,
                                                       const float* __restrict__ XHt, double* __restrict__ viol_partial) {
  extern __shared__ double wrow_all[];  // [WARPS][f]
  __shared__ double vpart[WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * WARPS + warp;
  double* wr = wrow_all + (size_t)warp * f;
  double viol = 0.0;
  if (row < n_rows) {
    float* ar = A + (size_t)row * f;
    const float* xr = XHt + (size_t)row * f;
    for (int c = lane; c < f; c += 32) wr[c] = ar[c];
    __syncwarp();
    for (int t = 0; t < f; ++t) {
      const double* h = HHt + (size_t)t * f;
      double g = 0.0;
      for (int r = lane; r < f; r += 32) g += h[r] * wr[r];
      const double grad = warp_sum(g) - (double)xr[t];
      const double wt = wr[t];
      const double pg = wt == 0.0 ? fmin(0.0, grad) : grad;
      viol += fabs(pg);
      const double hess = h[t];
      __syncwarp();
      if (lane == 0 && hess != 0.0) wr[t] = fmax(wt - grad / hess, 0.0);
      __syncwarp();
    }
    for (int c = lane; c < f; c += 32) ar[c] = (float)wr[c];
  }
  if (lane == 0) vpart[warp] = viol;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int w = 0; w < WARPS; ++w) v += vpart[w];
    viol_partial[blockIdx.x] = v;
  }
}

// partials[block] = sum over the block's grid-stride share of a[i] * b[i] (b NULL: a[i])
template <typename TA, typename TB>
__global__ void __launch_bounds__(256) dot_partial_kernel(long long n, const TA* __restrict__ a, const TB* __restrict__ b,
                                                          double* __restrict__ partials) {
  __shared__ double part[WARPS];
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += b ? (double)a[i] * (double)b[i] : (double)a[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < WARPS; ++w) s += part[w];
    partials[blockIdx.x] = s;
  }
}

// out[0] = sum of partials[0 .. n) (one block, fixed order)
__global__ void __launch_bounds__(256) sum_partials_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  __shared__ double part[WARPS];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < WARPS; ++w) s += part[w];
    out[0] = s;
  }
}

// slots: [0] result  [1] ||X||^2  [2] tr(W^T W . H H^T)  [3] tr(W^T X H^T)  [4] KL sum over non-zeros  [5] sum(WH)
//        [6] violation of the W step  [7] violation of the H step
enum { S_OUT = 0, S_NORMX, S_TRACE, S_CROSS, S_KLNZ, S_SUMWH, S_VW, S_VH, N_SLOTS };

__global__ void combine_kernel(int mode, double* s) {
  if (mode == 0) s[S_OUT] = (s[S_NORMX] + s[S_TRACE] - 2.0 * s[S_CROSS]) / 2.0;  // _beta_divergence, beta = 2, sparse X
  else if (mode == 1) s[S_OUT] = s[S_KLNZ] + s[S_SUMWH];                        // beta = 1
  else if (mode == 2) s[S_OUT] = s[S_VW];
  else s[S_OUT] = s[S_VW] + s[S_VH];
}

struct Csr {
  int n_rows;
  const int* ptr;
  const int* idx;
  const float* val;
};

struct Solver {
  cudaStream_t st;
  int f;
  Csr X, Xt;
  float* W;
  float* Ht;
  int n_max;
  DevBuf<float> num;
  DevBuf<double> Gw, Gh, split_part, cw, ch, row_loss, partials, slots;

  Solver(cudaStream_t s, int f_, Csr x, Csr xt, float* w, float* ht) : st(s), f(f_), X(x), Xt(xt), W(w), Ht(ht) {
    n_max = std::max(X.n_rows, Xt.n_rows);
    const int tiles = (f + 31) / 32;
    // the Grams and column sums run over both row counts, each with its own split count
    const size_t splits_gram = std::max(n_splits(X.n_rows, tiles * tiles), n_splits(Xt.n_rows, tiles * tiles));
    const size_t splits_col = std::max(n_splits(X.n_rows, tiles), n_splits(Xt.n_rows, tiles));
    num.alloc((size_t)n_max * f);
    Gw.alloc((size_t)f * f);
    Gh.alloc((size_t)f * f);
    split_part.alloc(std::max(splits_gram * f * f, splits_col * f));
    cw.alloc(f);
    ch.alloc(f);
    row_loss.alloc(X.n_rows);
    partials.alloc(std::max<size_t>(DOT_BLOCKS, div_up(n_max, WARPS)));
    slots.alloc(N_SLOTS);
    B200_CUDA(cudaMemsetAsync(slots.get(), 0, sizeof(double) * N_SLOTS, st));
  }

  void spmm(const Csr& A, const float* M, float* out) {
    spmm_kernel<<<div_up(A.n_rows, WARPS), 256, 0, st>>>(A.n_rows, A.ptr, A.idx, A.val, M, f, out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  void gram(const float* M, int n, double* G) {
    const int tiles = (f + 31) / 32;
    const int per = split_rows(n, tiles * tiles);
    const int splits = (int)div_up(n, per);
    B200_REQUIRE((size_t)splits * f * f <= split_part.n, "b200_nmf: Gram split workspace too small (%d splits)", splits);
    gram_partial_kernel<<<dim3(tiles * tiles, splits), 256, 0, st>>>(n, f, M, per, split_part.get());
    sum_splits_kernel<<<div_up((long long)f * f, 256), 256, 0, st>>>(split_part.get(), splits, (long long)f * f, G);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  }
  void colsum(const float* M, int n, double* s) {
    const int tiles = (f + 31) / 32;
    const int per = split_rows(n, tiles);
    const int splits = (int)div_up(n, per);
    B200_REQUIRE((size_t)splits * f <= split_part.n, "b200_nmf: column-sum split workspace too small (%d splits)", splits);
    colsum_partial_kernel<<<dim3(tiles, splits), 256, 0, st>>>(n, f, M, per, split_part.get());
    sum_splits_kernel<<<div_up(f, 256), 256, 0, st>>>(split_part.get(), splits, f, s);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  }
  template <typename TA, typename TB>
  void dot(long long n, const TA* a, const TB* b, int slot) {
    const int blocks = (int)std::min<long long>(DOT_BLOCKS, std::max<long long>(1, div_up(n, 256)));
    dot_partial_kernel<TA, TB><<<blocks, 256, 0, st>>>(n, a, b, partials.get());
    sum_partials_kernel<<<1, 256, 0, st>>>(partials.get(), blocks, slots.get() + slot);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  }
  void mu_fro(float* A, int n, const double* G) {
    const size_t bytes = 32 * 32 * sizeof(double) + (size_t)TR * f * sizeof(float);
    B200_CUDA(cudaFuncSetAttribute(mu_fro_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    mu_fro_update_kernel<<<div_up(n, TR), 256, bytes, st>>>(n, f, A, num.get(), G);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  void kl(const Csr& A_csr, float* A, const float* B, const double* s, int zero_to_one, int zero_small) {
    kl_kernel<<<div_up(A_csr.n_rows, WARPS), 256, 0, st>>>(A_csr.n_rows, A_csr.ptr, A_csr.idx, A_csr.val, A, B, f, s, zero_to_one,
                                                           zero_small, row_loss.get());
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  void cd(float* A, int n, const double* G, int slot) {
    const int blocks = (int)div_up(n, WARPS);
    cd_sweep_kernel<<<blocks, 256, (size_t)WARPS * f * sizeof(double), st>>>(n, f, A, G, num.get(), partials.get());
    sum_partials_kernel<<<1, 256, 0, st>>>(partials.get(), blocks, slots.get() + slot);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  }
  double read_out(int mode) {
    combine_kernel<<<1, 1, 0, st>>>(mode, slots.get());
    B200_CUDA(cudaGetLastError());
    count_launch();
    double h = 0.0;
    B200_CUDA(cudaMemcpyAsync(&h, slots.get() + S_OUT, sizeof(double), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return h;
  }

  // _beta_divergence(X, W, H, beta, square_root=True).  Frobenius: with fresh_h the X H^T (in num) and H H^T (in Gh) are
  // recomputed from Ht first; without it they are the ones the caller left there.
  double error(int beta_loss, bool fresh_h) {
    if (beta_loss == 0) {
      if (fresh_h) {
        gram(Ht, Xt.n_rows, Gh.get());
        spmm(X, Ht, num.get());
      }
      gram(W, X.n_rows, Gw.get());
      dot(1ll * f * f, Gw.get(), Gh.get(), S_TRACE);
      dot(1ll * X.n_rows * f, num.get(), W, S_CROSS);
      return std::sqrt(read_out(0) * 2.0);
    }
    colsum(W, X.n_rows, cw.get());
    colsum(Ht, Xt.n_rows, ch.get());
    dot(f, cw.get(), ch.get(), S_SUMWH);
    kl(X, W, Ht, nullptr, 0, 0);
    dot(X.n_rows, row_loss.get(), (const double*)nullptr, S_KLNZ);
    return std::sqrt(2.0 * std::max(read_out(1), 0.0));
  }

  // _fit_multiplicative_update with alpha_W = 0 (gamma = 1 for both losses)
  void mu(int beta_loss, bool update_h, int max_iter, double tol, int* n_iter, double* last_error) {
    if (beta_loss == 0 && !update_h) {  // H is fixed: X H^T and H H^T are computed once (update_H=False)
      gram(Ht, Xt.n_rows, Gh.get());
      spmm(X, Ht, num.get());
    }
    if (beta_loss == 1 && !update_h) colsum(Ht, Xt.n_rows, ch.get());
    double error_at_init = 0.0, previous = 0.0;
    if (tol > 0) {
      error_at_init = previous = error(beta_loss, update_h);
      *last_error = error_at_init;
    }
    int it = 1;
    for (; it <= max_iter; ++it) {
      if (beta_loss == 0) {
        if (update_h) {
          gram(Ht, Xt.n_rows, Gh.get());
          spmm(X, Ht, num.get());
        }
        mu_fro(W, X.n_rows, Gh.get());
        if (update_h) {
          gram(W, X.n_rows, Gw.get());
          spmm(Xt, W, num.get());
          mu_fro(Ht, Xt.n_rows, Gw.get());
        }
      } else {
        if (update_h) colsum(Ht, Xt.n_rows, ch.get());
        kl(X, W, Ht, ch.get(), 0, 0);
        if (update_h) {
          colsum(W, X.n_rows, cw.get());
          kl(Xt, Ht, W, cw.get(), 1, 1);
        }
      }
      if (tol > 0 && it % 10 == 0) {
        const double err = error(beta_loss, update_h);
        *last_error = err;
        if ((previous - err) / error_at_init < tol) break;
        previous = err;
      }
    }
    *n_iter = std::min(it, max_iter);
  }

  // _fit_coordinate_descent, shuffle=False, no regularisation
  void cd_solve(bool update_h, int max_iter, double tol, int* n_iter, double* last_error) {
    if (!update_h) {
      gram(Ht, Xt.n_rows, Gh.get());
      spmm(X, Ht, num.get());
    }
    double violation_init = 0.0;
    int it = 1;
    for (; it <= max_iter; ++it) {
      if (update_h) {
        gram(Ht, Xt.n_rows, Gh.get());
        spmm(X, Ht, num.get());
      }
      cd(W, X.n_rows, Gh.get(), S_VW);
      if (update_h) {
        gram(W, X.n_rows, Gw.get());
        spmm(Xt, W, num.get());
        cd(Ht, Xt.n_rows, Gw.get(), S_VH);
      }
      const double violation = read_out(update_h ? 3 : 2);
      *last_error = violation;
      if (it == 1) violation_init = violation;
      if (violation_init == 0.0) break;
      if (violation / violation_init <= tol) break;
    }
    *n_iter = std::min(it, max_iter);
  }
};

}  // namespace nmf
}  // namespace b200

using namespace b200;
using namespace b200::nmf;

extern "C" {

int b200_nmf_solve_device(int solver, int beta_loss, int update_h, int n_users, int n_items, int n_factors, const int32_t* d_x_ptr,
                          const int32_t* d_x_idx, const float* d_x_val, const int32_t* d_xt_ptr, const int32_t* d_xt_idx,
                          const float* d_xt_val, float* d_W, float* d_Ht, int max_iter, double tol, int32_t* n_iter,
                          double* last_error, void* stream) {
  return guarded([&] {
    B200_REQUIRE(solver == B200_NMF_MU || solver == B200_NMF_CD, "b200_nmf_solve: unknown solver %d", solver);
    B200_REQUIRE(beta_loss == B200_NMF_FROBENIUS || beta_loss == B200_NMF_KL, "b200_nmf_solve: unknown beta_loss %d", beta_loss);
    B200_REQUIRE(!(solver == B200_NMF_CD && beta_loss != B200_NMF_FROBENIUS),
                 "Invalid beta_loss parameter: solver 'cd' does not handle beta_loss = 'kullback-leibler'");
    B200_REQUIRE(n_users > 0 && n_items > 0 && n_factors >= 1 && n_factors <= F_MAX,
                 "b200_nmf_solve: bad shape (n_users %d, n_items %d, n_factors %d; 1 <= n_factors <= %d)", n_users, n_items,
                 n_factors, F_MAX);
    B200_REQUIRE(d_x_ptr && d_x_idx && d_x_val && d_W && d_Ht && n_iter && last_error, "b200_nmf_solve: NULL argument");
    B200_REQUIRE(!update_h || (d_xt_ptr && d_xt_idx && d_xt_val), "b200_nmf_solve: the fit needs the CSR of X^T");
    B200_REQUIRE(max_iter >= 1 && tol >= 0, "b200_nmf_solve: bad max_iter / tol");
    // X^T is only read by the H step; transform passes the item count alone (rows of Ht)
    Solver s((cudaStream_t)stream, n_factors, Csr{n_users, d_x_ptr, d_x_idx, d_x_val}, Csr{n_items, d_xt_ptr, d_xt_idx, d_xt_val},
             d_W, d_Ht);
    *last_error = 0.0;
    if (solver == B200_NMF_MU) {
      if (tol > 0 && beta_loss == B200_NMF_FROBENIUS) {
        int nnz = 0;
        B200_CUDA(cudaMemcpyAsync(&nnz, d_x_ptr + n_users, sizeof(int), cudaMemcpyDeviceToHost, s.st));
        B200_CUDA(cudaStreamSynchronize(s.st));
        s.dot((long long)nnz, d_x_val, d_x_val, S_NORMX);
      }
      s.mu(beta_loss, update_h != 0, max_iter, tol, n_iter, last_error);
    } else {
      s.cd_solve(update_h != 0, max_iter, tol, n_iter, last_error);
    }
    B200_CUDA(cudaStreamSynchronize(s.st));
  });
}

int b200_nmf_debug_device(int op, int n_rows, int n_factors, const int32_t* d_ptr, const int32_t* d_idx, const float* d_val,
                          const float* d_M, void* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n_rows > 0 && n_factors >= 1 && n_factors <= F_MAX && d_M && d_out, "b200_nmf_debug: bad argument");
    B200_REQUIRE(op == 1 || (op == 0 && d_ptr && d_idx && d_val), "b200_nmf_debug: bad op %d", op);
    Csr a{n_rows, d_ptr, d_idx, d_val};
    Solver s((cudaStream_t)stream, n_factors, a, a, nullptr, nullptr);
    if (op == 0) s.spmm(a, d_M, (float*)d_out);
    else s.gram(d_M, n_rows, (double*)d_out);
    B200_CUDA(cudaStreamSynchronize(s.st));
  });
}

}  // extern "C"
