// K7: SLIM ElasticNet -- one non-negative (optionally signed) elastic-net regression per item, on the Gram matrix, sm_90a.
//
// Replaces the per-item loop of SLIM_ElasticNet/SLIMElasticNetRecommender.py:77-131, i.e. scikit-learn's
// ElasticNet(precompute=True, fit_intercept=False, max_iter=100, tol=1e-4).fit(URM with column j zeroed, URM[:, j]) -- the
// Gram-matrix coordinate descent `enet_coordinate_descent_gram` (restated in oracle/elasticnet_oracle.py with its stopping
// rule: a pass with max|dw| / max|w| < tol triggers the duality gap, the solve ends when gap < tol * ||y||^2).
//
// The reference fits the items one after the other and recomputes X^T X for every item; here the Gram matrix G is computed
// ONCE on the device (K1's dense mode, as for EASE_R) and every CTA solves one item at a time against it:
//   Q = G with row / column j removed (the target column is zeroed, :88), q = G[:, j], ||y||^2 = G[j, j].
// Coordinate descent is sequential in the coordinates, but a coordinate whose weight is 0 and stays 0 changes nothing
// (q_k - H_k <= l1), so the CTA scans the coordinates 512 at a time against the current H = Q w, finds the FIRST one that
// acts (per-warp ballots, one barrier), applies it (H += (new - old) * Q[k, :], one coalesced row of G, requested while thread 0
// still computes the new weight) and rescans from k + 1: exactly the cyclic sweep, at the cost of one row of G and three
// barriers per active coordinate.  w, H and q live in shared memory up to 3 * n * 4 bytes <= 200 KB (C4: 17.7 K
// items = 208 KB), in an L2-resident workspace beyond that.
// The reference draws the coordinate order at random from an unseeded generator; the cyclic order reaches the same optimum
// within the same tolerance (tests/test_oracle_elasticnet.py pins that against the reference's own output).
// Roofline: L2 bandwidth -- (active coordinates x passes) rows of G per item.
#include <algorithm>

#include "common.cuh"

namespace b200 {
namespace enet {

constexpr int THREADS = 512;
constexpr int WARPS = THREADS / 32;
constexpr int PRE = 8;  // elements of a row of G a thread requests before the step is known

struct Params {
  const float* __restrict__ G;     // [n, n] symmetric; the diagonal is taken from diag
  const float* __restrict__ diag;  // [n] sum of squares of every column of the URM
  int n, positive, max_iter;
  float l1, l2, tol;
  float* coefT;                    // [n, n]: row j = the coefficients of the model of item j
  int* n_iter;                     // nullable [n]
  float* work;                     // nullable: gridDim.x * 3 * n floats when the vectors do not fit shared memory
  int* counter;
};

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < WARPS; ++w) t += red[w];
  return t;
}
__device__ __forceinline__ float block_max(float v, double* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = (double)v;
  __syncthreads();
  float t = (float)red[0];
#pragma unroll
  for (int w = 1; w < WARPS; ++w) t = fmaxf(t, (float)red[w]);
  return t;
}

__global__ void __launch_bounds__(THREADS) slim_enet_kernel(const Params p) {
  extern __shared__ float sm[];
  __shared__ double red[WARPS];
  __shared__ int s_item;
  __shared__ unsigned s_ballot[WARPS];
  __shared__ float s_old, s_new, s_wmax, s_dwmax;
  const int n = p.n, tid = threadIdx.x, lane = tid & 31;
  float* w = p.work ? p.work + (size_t)blockIdx.x * 3 * n : sm;
  float* H = w + n;
  float* q = H + n;
  for (;;) {
    __syncthreads();
    if (tid == 0) s_item = atomicAdd(p.counter, 1);
    __syncthreads();
    const int j = s_item;
    if (j >= n) break;
    const float* Gj = p.G + (size_t)j * n;
    const float y_norm2 = p.diag[j];
    for (int c = tid; c < n; c += THREADS) { w[c] = 0.f; H[c] = 0.f; q[c] = c == j ? 0.f : Gj[c]; }
    __syncthreads();
    int it = 0;
    if (y_norm2 > 0.f) {
      const float tol_gap = p.tol * y_norm2;
      for (it = 1; it <= p.max_iter; ++it) {
        if (tid == 0) { s_wmax = 0.f; s_dwmax = 0.f; }
        // ---- one cyclic pass: find the next coordinate that acts, apply it, go on behind it
        int k0 = 0;
        while (k0 < n) {
          const int k = k0 + tid;
          bool acts = false;
          if (k < n && k != j) {
            const float d = p.diag[k];
            if (d != 0.f) {  // Q[ii, ii] == 0: skipped
              const float wk = w[k];
              if (wk != 0.f) acts = true;
              else {
                const float tmp = q[k] - H[k];
                acts = p.positive ? tmp > p.l1 : fabsf(tmp) > p.l1;
              }
            }
          }
          const unsigned b = __ballot_sync(0xffffffffu, acts);
          if (lane == 0) s_ballot[tid >> 5] = b;
          if (!__syncthreads_or(acts)) { k0 += THREADS; continue; }  // also publishes the ballots
          int kf = k0;
#pragma unroll
          for (int wv = WARPS - 1; wv >= 0; --wv) {  // the lowest acting coordinate of the chunk
            const unsigned bw = s_ballot[wv];
            if (bw) kf = k0 + wv * 32 + __ffs(bw) - 1;
          }
          // its row of G is requested before the new weight is known (PRE values per thread stay in registers)
          const float* Gk = p.G + (size_t)kf * n;
          float gpre[PRE];
#pragma unroll
          for (int m = 0; m < PRE; ++m) {
            const int c = tid + m * THREADS;
            gpre[m] = c < n ? Gk[c] : 0.f;
          }
          if (tid == 0) {
            const float d = p.diag[kf], wk = w[kf];
            float hk = H[kf];
            if (wk != 0.f) hk -= wk * d;
            const float tmp = q[kf] - hk;
            float nw;
            if (p.positive && tmp < 0.f) nw = 0.f;
            else nw = copysignf(fmaxf(fabsf(tmp) - p.l1, 0.f), tmp) / (d + p.l2);
            w[kf] = nw;
            s_old = wk; s_new = nw;
            s_dwmax = fmaxf(s_dwmax, fabsf(nw - wk));
            s_wmax = fmaxf(s_wmax, fabsf(nw));
          }
          __syncthreads();
          const float wk = s_old, nw = s_new;
          if (wk != nw) {
            const float dk = p.diag[kf];
#pragma unroll
            for (int m = 0; m < PRE; ++m) {
              const int c = tid + m * THREADS;
              if (c < n && c != j) {  // column j of Q is zero
                const float g = c == kf ? dk : gpre[m];
                float h = H[c];
                h -= wk * g;
                h += nw * g;
                H[c] = h;
              }
            }
            for (int c = tid + PRE * THREADS; c < n; c += THREADS) {
              if (c == j) continue;
              const float g = c == kf ? dk : Gk[c];
              float h = H[c];
              h -= wk * g;
              h += nw * g;
              H[c] = h;
            }
          }
          k0 = kf + 1;
          __syncthreads();
        }
        __syncthreads();
        const float w_max = s_wmax, d_w_max = s_dwmax;
        __syncthreads();  // the next pass resets them
        if (w_max == 0.f || d_w_max / w_max < p.tol || it == p.max_iter) {
          // duality gap of the elastic net on the Gram matrix
          double qw = 0.0, wHw = 0.0, ww = 0.0, l1n = 0.0;
          float xta = -3.4e38f;
          for (int c = tid; c < n; c += THREADS) {
            const float wc = w[c], hc = H[c], qc = q[c];
            qw += (double)wc * qc; wHw += (double)wc * hc; ww += (double)wc * wc; l1n += fabs((double)wc);
            const float x = qc - hc - p.l2 * wc;
            xta = fmaxf(xta, p.positive ? x : fabsf(x));
          }
          qw = block_sum(qw, red); wHw = block_sum(wHw, red); ww = block_sum(ww, red); l1n = block_sum(l1n, red);
          const double dual = (double)block_max(xta, red);
          const double R = (double)y_norm2 + wHw - 2.0 * qw;
          double cst, gap;
          if (dual > (double)p.l1) { cst = (double)p.l1 / dual; gap = 0.5 * (R + R * cst * cst); }
          else { cst = 1.0; gap = R; }
          gap += (double)p.l1 * l1n - cst * (double)y_norm2 + cst * qw + 0.5 * (double)p.l2 * (1.0 + cst * cst) * ww;
          if (gap < (double)tol_gap) break;  // uniform: every thread holds the same sums
        }
      }
      if (it > p.max_iter) it = p.max_iter;
    }
    float* out = p.coefT + (size_t)j * n;
    for (int c = tid; c < n; c += THREADS) out[c] = w[c];
    if (tid == 0 && p.n_iter) p.n_iter[j] = it;
  }
}

}  // namespace enet
}  // namespace b200

using namespace b200;
using namespace b200::enet;

extern "C" {

int b200_slim_enet_device(const float* d_G, const float* d_diag, int n_items, int64_t n_users, double l1_ratio, double alpha,
                          int positive_only, int max_iter, float tol, float* d_coef_T, int32_t* d_n_iter, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_G && d_diag && d_coef_T, "b200_slim_enet: NULL argument");
    B200_REQUIRE(n_items > 0 && n_users > 0 && max_iter > 0 && tol > 0.f, "b200_slim_enet: bad shape / max_iter / tol");
    B200_REQUIRE(l1_ratio >= 0.0 && l1_ratio <= 1.0, "b200_slim_enet: l1_ratio must be between 0 and 1, provided value was %g", l1_ratio);
    cudaStream_t st = (cudaStream_t)stream;
    Params p{};
    p.G = d_G; p.diag = d_diag; p.n = n_items; p.positive = positive_only != 0; p.max_iter = max_iter; p.tol = tol;
    p.l1 = (float)(alpha * l1_ratio * (double)n_users);          // sklearn: l1_reg = alpha * l1_ratio * n_samples
    p.l2 = (float)(alpha * (1.0 - l1_ratio) * (double)n_users);  //          l2_reg = alpha * (1 - l1_ratio) * n_samples
    p.coefT = d_coef_T; p.n_iter = d_n_iter;
    const size_t vec_bytes = (size_t)3 * (size_t)n_items * sizeof(float);
    const int grid = std::min(n_items, sm_count());
    DevBuf<float> work;
    DevBuf<int> counter(1);
    B200_CUDA(cudaMemsetAsync(counter.get(), 0, sizeof(int), st));
    p.counter = counter.get();
    size_t smem = vec_bytes;
    if (vec_bytes > 200 * 1024) {
      work.alloc((size_t)grid * 3 * (size_t)n_items);
      p.work = work.get();
      smem = 0;
    }
    B200_CUDA(cudaFuncSetAttribute(slim_enet_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1024)));
    slim_enet_kernel<<<grid, THREADS, smem, st>>>(p);
    B200_CUDA(cudaGetLastError());
    count_launch();
    B200_CUDA(cudaStreamSynchronize(st));  // the counter / workspace are released on return
  });
}

}  // extern "C"
