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
//
// Sparse Gram (large catalogues, positive_only on a non-negative URM): G as a CSR without its diagonal, and no n x n
// buffer.  There G >= 0 and w >= 0, so H_k = (Q w)_k >= 0, and a coordinate k with G[j, k] = 0 has q_k = 0 and
// q_k - H_k <= 0 <= l1: it never acts.  The solve of item j therefore scans only the support of row j of G (ascending, so
// the same coordinates act in the same order) and an applied coordinate k updates H over the non-zeros of row k only, with
// the dense path's expressions.  w, H and q are read on the support alone, so each item resets them there and nowhere
// else (entries outside it are written by the row updates but never read).  When the item ends, its min(nnz - 1, K) largest
// weights go straight into an [n, K] top-K table (dense_topk.cu's mode 2): no coefficient line is stored.
#include <algorithm>

#include "common.cuh"
#include "select.cuh"

namespace b200 {
namespace enet {

constexpr int THREADS = 512;
constexpr int WARPS = THREADS / 32;
constexpr int PRE = 8;  // elements of a row of G a thread requests before the step is known
constexpr int BINS = 2048;  // the top-K select's 11-bit digits
constexpr size_t SMEM_VECTORS = 200 * 1024;  // w, H and q in shared memory up to this size, in the workspace beyond it

struct Params {
  const float* __restrict__ G;        // dense: [n, n] symmetric, the diagonal is taken from diag; sparse: the CSR values
  const long long* __restrict__ gptr;  // sparse: [n + 1] row starts of the CSR
  const int* __restrict__ gcol;        // sparse: ascending column ids per row, the diagonal not stored
  const float* __restrict__ diag;  // [n] sum of squares of every column of the URM
  int n, positive, max_iter;
  float l1, l2, tol;
  float* coefT;                    // dense: [n, n], row j = the coefficients of the model of item j
  int K;                           // sparse: the top-K table [n, K] (top_idx = -1 / top_val = 0 past top_cnt)
  int* top_idx;
  float* top_val;
  int* top_cnt;
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

// H[c] after coordinate k moved from wk to nw (g = Q[k, c]); both paths write it this way, so that it contracts alike
__device__ __forceinline__ void update_h(float* H, int c, float wk, float nw, float g) {
  float h = H[c];
  h -= wk * g;
  h += nw * g;
  H[c] = h;
}

// Item j's [K] row of the top-K table: the min(nnz - 1, K) largest non-zero weights of the support sc[0, m), ties to
// the ascending index (dense_topk.cu's mode 2).
__device__ __forceinline__ void support_topk(int K, int* out_idx, float* out_val, int* out_cnt, const int* sc, int m,
                                             const float* w) {
  __shared__ CtaSelectSmem<BINS> sel;
  __shared__ int s_nnz, s_cnt, s_tie;
  const int tid = threadIdx.x;
  if (tid == 0) { s_nnz = 0; s_cnt = 0; s_tie = 0; }
  __syncthreads();
  int nnz = 0;
  for (int e = tid; e < m; e += THREADS) nnz += w[sc[e]] != 0.f;
  nnz = __reduce_add_sync(0xffffffffu, nnz);
  if ((tid & 31) == 0) atomicAdd(&s_nnz, nnz);
  __syncthreads();
  nnz = s_nnz;
  const int keep = drop_last_keep(K, nnz);
  u64 thr = 0;
  int ties = keep;
  if (keep > 0 && keep < nnz) {
    const auto key_at = [&](int e, u64& key) {
      const float v = w[sc[e]];
      if (v != 0.f) key = line_key(v, sc[e], false);
      return v != 0.f;
    };
    const Threshold<u64> t = radix_select<u64, 11, false>(CtaSelect<THREADS, BINS>(sel), m, keep, key_at);
    thr = t.thr;
    ties = t.need;
  }
  if (keep > 0) {
    for (int e = tid; e < m; e += THREADS) {
      const int c = sc[e];
      const float v = w[c];
      if (v != 0.f) {
        const u64 key = line_key(v, c, false);
        if (key > thr || (key == thr && atomicAdd(&s_tie, 1) < ties)) {
          const int pos = atomicAdd(&s_cnt, 1);
          out_idx[pos] = c;
          out_val[pos] = v;
        }
      }
    }
  }
  __syncthreads();
  const int cnt = s_cnt;
  for (int t = cnt + tid; t < K; t += THREADS) { out_idx[t] = -1; out_val[t] = 0.f; }
  if (tid == 0) *out_cnt = cnt;
}

// The solve loop of both kernels.  SPARSE: G is the CSR (gptr, gcol, G) and positive is 1 (see the head of the file).
template <bool SPARSE>
__device__ __forceinline__ void solve_items(const Params p) {
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
    // the coordinates item j visits, by position e in [0, m): every coordinate (dense), or the support of row j (sparse)
    const long long s0 = SPARSE ? p.gptr[j] : 0;
    const int m = SPARSE ? (int)(p.gptr[j + 1] - s0) : n;
    const int* sc = SPARSE ? p.gcol + s0 : nullptr;
    const float y_norm2 = p.diag[j];
    if (SPARSE) {
      for (int e = tid; e < m; e += THREADS) { const int c = sc[e]; w[c] = 0.f; H[c] = 0.f; q[c] = p.G[s0 + e]; }
    } else {
      const float* Gj = p.G + (size_t)j * n;
      for (int c = tid; c < n; c += THREADS) { w[c] = 0.f; H[c] = 0.f; q[c] = c == j ? 0.f : Gj[c]; }
    }
    __syncthreads();
    int it = 0;
    if (y_norm2 > 0.f) {
      const float tol_gap = p.tol * y_norm2;
      for (it = 1; it <= p.max_iter; ++it) {
        if (tid == 0) { s_wmax = 0.f; s_dwmax = 0.f; }
        // ---- one cyclic pass: find the next coordinate that acts, apply it, go on behind it
        int e0 = 0;
        while (e0 < m) {
          const int e = e0 + tid;
          bool acts = false;
          const int k = SPARSE ? (e < m ? sc[e] : j) : e;
          if (e < m && k != j) {
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
          if (!__syncthreads_or(acts)) { e0 += THREADS; continue; }  // also publishes the ballots
          int ef = e0;
#pragma unroll
          for (int wv = WARPS - 1; wv >= 0; --wv) {  // the lowest acting coordinate of the chunk
            const unsigned bw = s_ballot[wv];
            if (bw) ef = e0 + wv * 32 + __ffs(bw) - 1;
          }
          const int kf = SPARSE ? sc[ef] : ef;
          // its row of G is requested before the new weight is known (PRE values per thread stay in registers)
          const long long r0 = SPARSE ? p.gptr[kf] : (long long)kf * n;
          const int rl = SPARSE ? (int)(p.gptr[kf + 1] - r0) : n;
          const float* Gk = p.G + r0;
          const int* Ck = SPARSE ? p.gcol + r0 : nullptr;
          float gpre[PRE];
          int cpre[PRE];
#pragma unroll
          for (int mm = 0; mm < PRE; ++mm) {
            const int r = tid + mm * THREADS;
            gpre[mm] = r < rl ? Gk[r] : 0.f;
            cpre[mm] = SPARSE ? (r < rl ? Ck[r] : j) : r;
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
            for (int mm = 0; mm < PRE; ++mm) {
              const int c = cpre[mm];
              if (tid + mm * THREADS < rl && c != j)  // column j of Q is zero
                update_h(H, c, wk, nw, c == kf ? dk : gpre[mm]);
            }
            for (int r = tid + PRE * THREADS; r < rl; r += THREADS) {
              const int c = SPARSE ? Ck[r] : r;
              if (c == j) continue;
              update_h(H, c, wk, nw, c == kf ? dk : Gk[r]);
            }
            if (SPARSE && tid == 0) update_h(H, kf, wk, nw, dk);  // the CSR does not store the diagonal
          }
          e0 = ef + 1;
          __syncthreads();
        }
        __syncthreads();
        const float w_max = s_wmax, d_w_max = s_dwmax;
        __syncthreads();  // the next pass resets them
        if (w_max == 0.f || d_w_max / w_max < p.tol || it == p.max_iter) {
          // duality gap of the elastic net on the Gram matrix.  The dense maximum of XtA includes coordinate j, where
          // it is exactly 0; outside the support it is -H_k <= 0: the sparse maximum starts at 0 instead.
          double qw = 0.0, wHw = 0.0, ww = 0.0, l1n = 0.0;
          float xta = SPARSE ? 0.f : -3.4e38f;
          for (int e = tid; e < m; e += THREADS) {
            const int c = SPARSE ? sc[e] : e;
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
    if (SPARSE) {
      support_topk(p.K, p.top_idx + (size_t)j * p.K, p.top_val + (size_t)j * p.K, p.top_cnt + j, sc, m, w);
    } else {
      float* out = p.coefT + (size_t)j * n;
      for (int c = tid; c < n; c += THREADS) out[c] = w[c];
    }
    if (tid == 0 && p.n_iter) p.n_iter[j] = it;
  }
}

__global__ void __launch_bounds__(THREADS) slim_enet_kernel(const Params p) { solve_items<false>(p); }
// With the top-K select inlined, ptxas's default budget for 512 threads (64 registers) spills; 72 do not.  (More than
// 72 is no better: the dense loop spills at 80 and 96.)
__global__ void __maxnreg__(72) slim_enet_sparse_kernel(const Params p) { solve_items<true>(p); }

// Compaction of a slab of rows [row0, row0 + rows) of a dense [n, n] Gram matrix into CSR rows: one warp per row, 32
// columns per ballot, so the column ids come out ascending.  The diagonal is dropped (the solve reads it from diag).
constexpr int COMPACT_THREADS = 256;

template <bool FILL>
__global__ void __launch_bounds__(COMPACT_THREADS) gram_slab_compact_kernel(const float* __restrict__ S, int rows, int n, int row0,
                                                                            long long* __restrict__ row_nnz,
                                                                            const long long* __restrict__ row_start,
                                                                            int* __restrict__ col, float* __restrict__ val) {
  const int r = blockIdx.x * (COMPACT_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* Sr = S + (size_t)r * n;
  const int diag = row0 + r;
  long long pos = FILL ? row_start[r] : 0;
  const long long end = FILL ? row_start[r + 1] : 0;
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int c = c0 + lane;
    const float v = c < n ? Sr[c] : 0.f;
    const bool nz = v != 0.f && c != diag;
    const unsigned b = __ballot_sync(0xffffffffu, nz);
    if (FILL && nz) {
      const long long at = pos + __popc(b & ((1u << lane) - 1u));
      if (at < end) { col[at] = c; val[at] = v; }
    }
    pos += __popc(b);
  }
  if (!FILL && lane == 0) row_nnz[r] = pos;
}

size_t work_floats(int n_items, int grid) {
  const size_t vec_bytes = (size_t)3 * (size_t)n_items * sizeof(float);
  return vec_bytes > SMEM_VECTORS ? (size_t)grid * 3 * (size_t)n_items : 0;
}

template <class Kernel>
void launch(Kernel kernel, Params& p, int n_items, cudaStream_t st) {
  const int grid = std::min(n_items, sm_count());
  DevBuf<float> work;
  DevBuf<int> counter(1);
  B200_CUDA(cudaMemsetAsync(counter.get(), 0, sizeof(int), st));
  p.counter = counter.get();
  size_t smem = (size_t)3 * (size_t)n_items * sizeof(float);
  if (const size_t wf = work_floats(n_items, grid)) {
    work.alloc(wf);
    p.work = work.get();
    smem = 0;
  }
  B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1024)));
  kernel<<<grid, THREADS, smem, st>>>(p);
  B200_CUDA(cudaGetLastError());
  count_launch();
  B200_CUDA(cudaStreamSynchronize(st));  // the counter / workspace are released on return
}

void set_common(Params& p, const float* d_diag, int n_items, int64_t n_users, double l1_ratio, double alpha, int positive_only,
                int max_iter, float tol, int32_t* d_n_iter) {
  B200_REQUIRE(n_items > 0 && n_users > 0 && max_iter > 0 && tol > 0.f, "b200_slim_enet: bad shape / max_iter / tol");
  B200_REQUIRE(l1_ratio >= 0.0 && l1_ratio <= 1.0, "b200_slim_enet: l1_ratio must be between 0 and 1, provided value was %g", l1_ratio);
  p.diag = d_diag; p.n = n_items; p.positive = positive_only != 0; p.max_iter = max_iter; p.tol = tol;
  p.l1 = (float)(alpha * l1_ratio * (double)n_users);          // sklearn: l1_reg = alpha * l1_ratio * n_samples
  p.l2 = (float)(alpha * (1.0 - l1_ratio) * (double)n_users);  //          l2_reg = alpha * (1 - l1_ratio) * n_samples
  p.n_iter = d_n_iter;
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
    Params p{};
    set_common(p, d_diag, n_items, n_users, l1_ratio, alpha, positive_only, max_iter, tol, d_n_iter);
    p.G = d_G; p.coefT = d_coef_T;
    launch(slim_enet_kernel, p, n_items, (cudaStream_t)stream);
  });
}

int b200_slim_enet_sparse_device(const int64_t* d_gram_ptr, const int32_t* d_gram_col, const float* d_gram_val, const float* d_diag,
                                 int n_items, int64_t n_users, double l1_ratio, double alpha, int max_iter, float tol, int topK,
                                 int32_t* d_top_idx, float* d_top_val, int32_t* d_top_cnt, int32_t* d_n_iter, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_gram_ptr && d_gram_col && d_gram_val && d_diag && d_top_idx && d_top_val && d_top_cnt,
                 "b200_slim_enet_sparse: NULL argument");
    B200_REQUIRE(topK > 0 && topK <= n_items, "b200_slim_enet_sparse: need 0 < topK <= n_items (got %d, %d)", topK, n_items);
    Params p{};
    set_common(p, d_diag, n_items, n_users, l1_ratio, alpha, 1, max_iter, tol, d_n_iter);
    p.G = d_gram_val; p.gptr = reinterpret_cast<const long long*>(d_gram_ptr); p.gcol = d_gram_col;
    p.K = topK; p.top_idx = d_top_idx; p.top_val = d_top_val; p.top_cnt = d_top_cnt;
    launch(slim_enet_sparse_kernel, p, n_items, (cudaStream_t)stream);
  });
}

int b200_slim_enet_workspace_bytes(int n_items, int n_sms, int64_t* bytes) {
  return guarded([&] {
    B200_REQUIRE(n_items > 0 && n_sms > 0 && bytes, "b200_slim_enet_workspace_bytes: n_items and n_sms must be positive");
    *bytes = (int64_t)(work_floats(n_items, std::min(n_items, n_sms)) * sizeof(float));
  });
}

int b200_gram_slab_compact_device(const float* d_slab, int rows, int n, int row0, int64_t* d_row_nnz, const int64_t* d_row_start,
                                  int32_t* d_col, float* d_val, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_slab && rows > 0 && n > 0 && row0 >= 0 && row0 + rows <= n, "b200_gram_slab_compact: bad slab");
    B200_REQUIRE((d_row_nnz != nullptr) != (d_row_start != nullptr), "b200_gram_slab_compact: exactly one of d_row_nnz / d_row_start");
    B200_REQUIRE(!d_row_start || (d_col && d_val), "b200_gram_slab_compact: the fill pass needs d_col and d_val");
    const int grid = (rows + COMPACT_THREADS / 32 - 1) / (COMPACT_THREADS / 32);
    cudaStream_t st = (cudaStream_t)stream;
    if (d_row_start)
      gram_slab_compact_kernel<true><<<grid, COMPACT_THREADS, 0, st>>>(d_slab, rows, n, row0, nullptr,
                                                                       reinterpret_cast<const long long*>(d_row_start), d_col, d_val);
    else
      gram_slab_compact_kernel<false><<<grid, COMPACT_THREADS, 0, st>>>(d_slab, rows, n, row0, reinterpret_cast<long long*>(d_row_nnz),
                                                                        nullptr, nullptr, nullptr);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

}  // extern "C"
