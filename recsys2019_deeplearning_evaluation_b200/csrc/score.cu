// K6: batch scoring behind _compute_item_score / recommend, sm_90a.
//
// Replaces
//   Base/BaseSimilarityMatrixRecommender.py:73-92   item scores = URM[users] . W_sparse           (SpMM -> dense block)
//   Base/BaseSimilarityMatrixRecommender.py:97-116  user-based twin  W_sparse[users] . URM
//   Base/BaseMatrixFactorizationRecommender.py:38-70 scores = U[users] . V^T (+ biases)
//   Base/BaseRecommender.py:164-196                 seen items -> -inf, per-row top-`cutoff`
// Outputs are dense [B, n_items] fp32 blocks (the Evaluator asks for B <= 1000 users at a time,
// Base/Evaluation/Evaluator.py:422).  Roofline: HBM, dominated by the B*n_items*4 bytes written (+ read back by the
// mask / top-N passes) and, for the sparse product, 8 bytes per gathered (j, w) pair of W.
// The cand_* kernels score and rank per-user candidate lists instead (Evaluator.py:466-578, test items plus sampled
// negatives, ~100 per user): the work is proportional to the candidates, not to B * n_items.
// The mask and top-N kernels also take fp64 blocks: the evaluators rank the host score blocks of recommenders that are
// not this package's mirrors, and those often score in float64.
#include <algorithm>
#include <cfloat>

#include "common.cuh"
#include "select.cuh"

namespace b200 {
namespace score {

typedef unsigned long long u64;

// out[b, :] = sum over (i, r) in row users[b] of A:  r * Brow(i)   -- A, B both CSR; one CTA per output row
__global__ void __launch_bounds__(512) spmm_rows_kernel(const int* __restrict__ users, int n_users_block,
                                                        const int* __restrict__ a_ptr, const int* __restrict__ a_idx,
                                                        const float* __restrict__ a_val, const int* __restrict__ b_ptr,
                                                        const int* __restrict__ b_idx, const float* __restrict__ b_val,
                                                        int n_out_cols, float* out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  for (int b = blockIdx.x; b < n_users_block; b += gridDim.x) {
    float* o = out + (size_t)b * n_out_cols;
    for (int j = tid; j < n_out_cols; j += blockDim.x) o[j] = 0.f;
    __syncthreads();
    const int u = users[b];
    const int s = a_ptr[u], e = a_ptr[u + 1];
    for (int k = s + warp; k < e; k += nwarps) {
      const int i = a_idx[k];
      const float r = a_val[k];
      if (b_ptr) {
        for (int q = b_ptr[i] + lane; q < b_ptr[i + 1]; q += 32) atomicAdd(o + b_idx[q], r * b_val[q]);
      } else {  // dense B: row i is b_val[i * n_out_cols ..]
        const float* brow = b_val + (size_t)i * n_out_cols;
        for (int j = lane; j < n_out_cols; j += 32) atomicAdd(o + j, r * brow[j]);
      }
    }
    __syncthreads();
  }
}

// out[b, j] = U[users[b], :] . VT[:, j] (+ mu + bu[users[b]] + bi[j]);  VT is the transposed item-factor matrix
// [f, n_items] so that consecutive threads read consecutive items.  8 users per thread share every VT load.
constexpr int UT = 8;
__global__ void __launch_bounds__(256) mf_scores_kernel(const int* __restrict__ users, int n_users_block,
                                                        const float* __restrict__ U, const float* __restrict__ VT, int f,
                                                        int n_items, const float* __restrict__ bu, const float* __restrict__ bi,
                                                        const float* __restrict__ mu, float* out) {
  extern __shared__ float ush[];  // [UT][f]
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b0 = blockIdx.y * UT;
  for (int t = threadIdx.x; t < UT * f; t += blockDim.x) {
    const int bb = b0 + t / f;
    ush[t] = bb < n_users_block ? U[(size_t)users[bb] * f + (t % f)] : 0.f;
  }
  __syncthreads();
  if (j >= n_items) return;
  float acc[UT];
#pragma unroll
  for (int k = 0; k < UT; ++k) acc[k] = 0.f;
  for (int q = 0; q < f; ++q) {
    const float v = VT[(size_t)q * n_items + j];
#pragma unroll
    for (int k = 0; k < UT; ++k) acc[k] += ush[k * f + q] * v;
  }
  const float base = mu ? mu[0] + bi[j] : 0.f;
#pragma unroll
  for (int k = 0; k < UT; ++k) {
    const int bb = b0 + k;
    if (bb < n_users_block) out[(size_t)bb * n_items + j] = acc[k] + base + (mu ? bu[users[bb]] : 0.f);
  }
}

// 32 x 32 tiles; the row tiles are walked grid-stride along y, whose grid size is capped at 65 535
__global__ void transpose_kernel(const float* __restrict__ in, int rows, int cols, float* out) {
  __shared__ float tile[32][33];
  const int x = blockIdx.x * 32 + threadIdx.x, oy0 = blockIdx.x * 32;
  for (int y0 = blockIdx.y * 32; y0 < rows; y0 += gridDim.y * 32) {
    for (int k = threadIdx.y; k < 32; k += blockDim.y)
      if (x < cols && y0 + k < rows) tile[k][threadIdx.x] = in[(size_t)(y0 + k) * cols + x];
    __syncthreads();
    const int ox = y0 + threadIdx.x;
    for (int k = threadIdx.y; k < 32; k += blockDim.y)
      if (ox < rows && oy0 + k < cols) out[(size_t)(oy0 + k) * rows + ox] = tile[threadIdx.x][k];
    __syncthreads();
  }
}

// scores[b, seen items of users[b]] = -inf (BaseRecommender.py:164-169); one warp per user
template <typename T>
__global__ void mask_seen_kernel(const int* __restrict__ users, int n_users_block, const int* __restrict__ ptr,
                                 const int* __restrict__ idx, int n_items, T* scores) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_users_block) return;
  const int u = users[warp];
  for (int k = ptr[u] + lane; k < ptr[u + 1]; k += 32) scores[(size_t)warp * n_items + idx[k]] = -INFINITY;
}

// items_to_compute (BaseSimilarityMatrixRecommender.py:80-86): every other item -> -inf.  keep[j] != 0 marks kept items.
template <typename T>
__global__ void mask_items_kernel(const unsigned char* __restrict__ keep, int n_users_block, int n_items, T* scores) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n_users_block * n_items) return;
  if (!keep[g % n_items]) scores[g] = -INFINITY;
}

// Unsigned key in the order of np.lexsort((arange, -s)), the host ranking (BaseRecommender.py:189-196): +inf, finite
// values descending, -inf, then NaN of either sign (key 0, below -inf's 0x007FFFFF).  -0 and +0 are one value, so they
// tie and fall back to the item index.
__device__ __forceinline__ unsigned lexsort_order(float v) { return v != v ? 0u : orderable(v == 0.f ? 0.f : v); }
// the same order on doubles: NaN -> 0, below -inf's 0x000FFFFFFFFFFFFF
__device__ __forceinline__ u64 lexsort_order(double v) { return v != v ? 0ull : orderable(v == 0.0 ? 0.0 : v); }

// The top-N key of the score at position q: the lexsort order of the score, then ~q, so that larger keys rank first and
// equal scores go to the lower position.  fp32: one 64-bit word, 6 radix passes of 11 bits.  fp64: 96 bits, 9 passes.
// `image` is what the table reports for a score: fp32 as it is; fp64 rounded to fp32 with finite values saturated to
// +-FLT_MAX, so that an entry is finite exactly when its score is (the evaluation kernels read nothing else).
template <typename T> struct TopnKey;
template <> struct TopnKey<float> {
  typedef u64 Key;
  static __device__ __forceinline__ Key make(float v, int q) { return KeyBits<Key>::make(lexsort_order(v), 0xFFFFFFFFu - (unsigned)q); }
  static __device__ __forceinline__ float image(float v) { return v; }
};
template <> struct TopnKey<double> {
  typedef Key96 Key;
  static __device__ __forceinline__ Key make(double v, int q) { return KeyBits<Key>::make(lexsort_order(v), 0xFFFFFFFFu - (unsigned)q); }
  static __device__ __forceinline__ float image(double v) {
    const float f = (float)v;
    return isfinite(v) ? fminf(fmaxf(f, -FLT_MAX), FLT_MAX) : f;
  }
};

// The `cutoff` best of the n scores L[0..n) of one row, best first (BaseRecommender.py:189-196); ties -> ascending
// position.  Position q is item q, or items[q] when a (strictly ascending) item map is given, so that ties go to the
// ascending item either way.  Called by all TOPN_THREADS threads of a CTA: radix select of the cutoff-th TopnKey key
// (select.cuh, 11-bit digits), then the survivors are ranked by counting (cutoff is small: <= 1024).
// out_items / out_scores: this row's `cutoff` slots; past the end of the row -1 / -inf.
constexpr int TOPN_THREADS = 256;
constexpr int TOPN_MAX = 1024;
template <typename T>
struct TopnSmem {
  CtaSelectSmem<2048> sel;
  int cnt;
  typename TopnKey<T>::Key cand[TOPN_MAX];
};
template <typename T>
__device__ __forceinline__ void topn_row(const T* L, int n, int cutoff, const int* items, int* out_items, float* out_scores,
                                         TopnSmem<T>& sm) {
  typedef TopnKey<T> K;
  typedef typename K::Key Key;
  typedef KeyBits<Key> KB;
  const int tid = threadIdx.x;
  const int keep = min(cutoff, n);
  Key thr{};
  if (keep < n) {
    const auto sel_key = [&](int q, Key& key) {
      key = K::make(L[q], q);
      return true;
    };
    thr = radix_select<Key, 11, false>(CtaSelect<TOPN_THREADS, 2048>(sm.sel), n, keep, sel_key).thr;
  }
  if (tid == 0) sm.cnt = 0;
  __syncthreads();
  for (int q = tid; q < n; q += TOPN_THREADS) {
    const Key key = K::make(L[q], q);
    if (KB::at_least(key, thr)) sm.cand[atomicAdd(&sm.cnt, 1)] = key;
  }
  __syncthreads();
  const int m = sm.cnt;  // == keep
  for (int t = tid; t < m; t += TOPN_THREADS) {
    const Key k = sm.cand[t];
    int rank = 0;
    for (int q = 0; q < m; ++q) rank += KB::greater(sm.cand[q], k);
    const int q = (int)(0xFFFFFFFFu - KB::low(k));
    out_items[rank] = items ? items[q] : q;
    out_scores[rank] = K::image(L[q]);
  }
  for (int t = m + tid; t < cutoff; t += TOPN_THREADS) { out_items[t] = -1; out_scores[t] = -INFINITY; }
  __syncthreads();
}

// per row of a dense [n_rows, n_items] block the `cutoff` best items; one CTA per row
template <typename T>
__global__ void __launch_bounds__(TOPN_THREADS) topn_rows_kernel(const T* __restrict__ scores, int n_rows, int n_items,
                                                                int cutoff, int* out_items, float* out_scores) {
  __shared__ TopnSmem<T> sm;
  for (int row = blockIdx.x; row < n_rows; row += gridDim.x)
    topn_row(scores + (size_t)row * n_items, n_items, cutoff, nullptr, out_items + (size_t)row * cutoff,
             out_scores + (size_t)row * cutoff, sm);
}

// ---- candidate lists (EvaluatorNegativeItemSample, Evaluator.py:466-578): every user is ranked over her own sorted list
// of candidate items only.  Row b of a block holds cand_idx[cand_ptr[b] .. cand_ptr[b + 1]); a per-candidate array is
// ragged, [cand_ptr[n_block] - cand_ptr[0]], entry k of the block at k - cand_ptr[0].  Every other item of the catalogue
// scores -inf on the full-catalogue path, so ranking the candidates alone gives the same +inf / finite prefix.
constexpr int CAND_THREADS = 256;
constexpr int CAND_STAGE = 2048;  // left-row entries staged in shared memory (16 KB); longer rows are read from global

__device__ __forceinline__ int lower_bound(const int* a, int n, int x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// score(b, c) = sum over j in row users[b] of A and column c of B of A[u, j] * B[j, c], column c of B being row c of
// (b_ptr, b_idx, b_val) with sorted indices: item-based A = URM, B rows = rows of W^T; user-based A = W, B rows = URM
// columns (CSC).  One CTA per user, the row of A staged in shared memory, one warp per candidate: the lanes walk the
// shorter of the two sorted lists and binary-search the longer one.
__global__ void __launch_bounds__(CAND_THREADS) cand_sparse_kernel(const int* __restrict__ users, const int* __restrict__ a_ptr,
                                                                  const int* __restrict__ a_idx, const float* __restrict__ a_val,
                                                                  const int* __restrict__ b_ptr, const int* __restrict__ b_idx,
                                                                  const float* __restrict__ b_val, const int* __restrict__ cand_ptr,
                                                                  const int* __restrict__ cand_idx, float* __restrict__ out) {
  __shared__ int s_idx[CAND_STAGE];
  __shared__ float s_val[CAND_STAGE];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int b = blockIdx.x, u = users[b];
  const int as = a_ptr[u], na = a_ptr[u + 1] - as;
  const int* ri = a_idx + as;
  const float* rv = a_val + as;
  if (na <= CAND_STAGE) {
    for (int t = tid; t < na; t += blockDim.x) { s_idx[t] = ri[t]; s_val[t] = rv[t]; }
    ri = s_idx;
    rv = s_val;
  }
  __syncthreads();
  const int base = cand_ptr[0], ce = cand_ptr[b + 1];
  for (int k = cand_ptr[b] + warp; k < ce; k += nwarps) {
    const int c = cand_idx[k];
    const int bs = b_ptr[c], nb = b_ptr[c + 1] - bs;
    const int* ci = b_idx + bs;
    const float* cv = b_val + bs;
    float acc = 0.f;
    if (nb <= na) {
      for (int q = lane; q < nb; q += 32) {
        const int j = ci[q], p = lower_bound(ri, na, j);
        if (p < na && ri[p] == j) acc += rv[p] * cv[q];
      }
    } else {
      for (int p = lane; p < na; p += 32) {
        const int j = ri[p], q = lower_bound(ci, nb, j);
        if (q < nb && ci[q] == j) acc += rv[p] * cv[q];
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) out[k - base] = acc;
  }
}

// score(b, c) = sum over (j, r) in row users[b] of A of r * B[j, c], B dense row-major [*, n_items] (EASE_R's dense W).
// One CTA per user, the row of A staged in shared memory, one thread per candidate summing in profile order.
__global__ void __launch_bounds__(CAND_THREADS) cand_dense_kernel(const int* __restrict__ users, const int* __restrict__ a_ptr,
                                                                 const int* __restrict__ a_idx, const float* __restrict__ a_val,
                                                                 const float* __restrict__ B, int n_items,
                                                                 const int* __restrict__ cand_ptr, const int* __restrict__ cand_idx,
                                                                 float* __restrict__ out) {
  __shared__ int s_idx[CAND_STAGE];
  __shared__ float s_val[CAND_STAGE];
  const int tid = threadIdx.x;
  const int b = blockIdx.x, u = users[b];
  const int as = a_ptr[u], na = a_ptr[u + 1] - as;
  const int* ri = a_idx + as;
  const float* rv = a_val + as;
  if (na <= CAND_STAGE) {
    for (int t = tid; t < na; t += blockDim.x) { s_idx[t] = ri[t]; s_val[t] = rv[t]; }
    ri = s_idx;
    rv = s_val;
  }
  __syncthreads();
  const int base = cand_ptr[0], ce = cand_ptr[b + 1];
  for (int k = cand_ptr[b] + tid; k < ce; k += blockDim.x) {
    const int c = cand_idx[k];
    float acc = 0.f;
    for (int p = 0; p < na; ++p) acc += rv[p] * B[(size_t)ri[p] * n_items + c];
    out[k - base] = acc;
  }
}

// score(b, c) = U[users[b], :] . V[c, :] (+ biases), one thread per (user, candidate) in the fp32 operation order of
// mf_scores_kernel (a sequential fused sum over the factors, then + (mu + bi) + bu), so the scores are bitwise those of the
// dense block.  One CTA per user, its factor row in shared memory; V row-major [n_items, f].
__global__ void __launch_bounds__(CAND_THREADS) cand_mf_kernel(const int* __restrict__ users, const float* __restrict__ U,
                                                              const float* __restrict__ V, int f, const float* __restrict__ bu,
                                                              const float* __restrict__ bi, const float* __restrict__ mu,
                                                              const int* __restrict__ cand_ptr, const int* __restrict__ cand_idx,
                                                              float* __restrict__ out) {
  extern __shared__ float us[];  // [f]
  const int tid = threadIdx.x;
  const int b = blockIdx.x, u = users[b];
  for (int t = tid; t < f; t += blockDim.x) us[t] = U[(size_t)u * f + t];
  __syncthreads();
  const int base = cand_ptr[0], ce = cand_ptr[b + 1];
  for (int k = cand_ptr[b] + tid; k < ce; k += blockDim.x) {
    const int c = cand_idx[k];
    const float* v = V + (size_t)c * f;
    float acc = 0.f;
    for (int q = 0; q < f; ++q) acc += us[q] * v[q];
    const float bias = mu ? mu[0] + bi[c] : 0.f;
    out[k - base] = acc + bias + (mu ? bu[u] : 0.f);
  }
}

// out[k] = scores[b, cand_idx[k]] from a dense [n_block, n_items] block; one warp per row
__global__ void cand_gather_kernel(int n_block, const float* __restrict__ scores, int n_items, const int* __restrict__ cand_ptr,
                                   const int* __restrict__ cand_idx, float* __restrict__ out) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (b >= n_block) return;
  const int base = cand_ptr[0], ce = cand_ptr[b + 1];
  for (int k = cand_ptr[b] + lane; k < ce; k += 32) out[k - base] = scores[(size_t)b * n_items + cand_idx[k]];
}

// BaseRecommender.py:164-169, :192-193: a seen candidate (binary search in the user's sorted train row) or an ignored one
// scores -inf
__device__ __forceinline__ float cand_masked(float v, int item, const int* seen, int n_seen, const unsigned char* ignore) {
  if (ignore && ignore[item]) return -INFINITY;
  if (n_seen > 0) {
    const int p = lower_bound(seen, n_seen, item);
    if (p < n_seen && seen[p] == item) return -INFINITY;
  }
  return v;
}

// candidate top-N, lists of up to CAND_WARP_LIST: one warp per user, keys in shared memory, rank by counting
constexpr int CAND_WARP_LIST = 256;
constexpr int CAND_TOPN_WARPS = 8;
__global__ void __launch_bounds__(CAND_TOPN_WARPS * 32) cand_topn_warp_kernel(
    const int* __restrict__ users, int n_block, const int* __restrict__ cand_ptr, const int* __restrict__ cand_idx,
    const float* __restrict__ scores, const int* __restrict__ seen_ptr, const int* __restrict__ seen_idx,
    const unsigned char* __restrict__ ignore, int cutoff, int* out_items, float* out_scores) {
  __shared__ u64 s_key[CAND_TOPN_WARPS][CAND_WARP_LIST];
  __shared__ float s_val[CAND_TOPN_WARPS][CAND_WARP_LIST];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * CAND_TOPN_WARPS + w;
  if (b >= n_block) return;
  const int cs = cand_ptr[b], n = cand_ptr[b + 1] - cs;
  if (n > CAND_WARP_LIST) return;  // cand_topn_cta_kernel's row
  const float* L = scores + (cs - cand_ptr[0]);
  const int* items = cand_idx + cs;
  const int* seen = nullptr;
  int n_seen = 0;
  if (seen_ptr) {
    const int u = users[b];
    seen = seen_idx + seen_ptr[u];
    n_seen = seen_ptr[u + 1] - seen_ptr[u];
  }
  for (int q = lane; q < n; q += 32) {
    const float v = cand_masked(L[q], items[q], seen, n_seen, ignore);
    s_val[w][q] = v;
    s_key[w][q] = TopnKey<float>::make(v, q);
  }
  __syncwarp();
  int* oi = out_items + (size_t)b * cutoff;
  float* os = out_scores + (size_t)b * cutoff;
  for (int q = lane; q < n; q += 32) {
    const u64 k = s_key[w][q];
    int rank = 0;
    for (int t = 0; t < n; ++t) rank += s_key[w][t] > k;
    if (rank < cutoff) { oi[rank] = items[q]; os[rank] = s_val[w][q]; }
  }
  for (int t = n + lane; t < cutoff; t += 32) { oi[t] = -1; os[t] = -INFINITY; }
}

// candidate top-N, lists longer than CAND_WARP_LIST: one CTA per user masks the scores in place, then topn_row
__global__ void __launch_bounds__(TOPN_THREADS) cand_topn_cta_kernel(
    const int* __restrict__ users, int n_block, const int* __restrict__ cand_ptr, const int* __restrict__ cand_idx,
    float* scores, const int* __restrict__ seen_ptr, const int* __restrict__ seen_idx, const unsigned char* __restrict__ ignore,
    int cutoff, int* out_items, float* out_scores) {
  __shared__ TopnSmem<float> sm;
  for (int b = blockIdx.x; b < n_block; b += gridDim.x) {
    const int cs = cand_ptr[b], n = cand_ptr[b + 1] - cs;
    if (n <= CAND_WARP_LIST) continue;
    float* L = scores + (cs - cand_ptr[0]);
    const int* items = cand_idx + cs;
    const int* seen = nullptr;
    int n_seen = 0;
    if (seen_ptr) {
      const int u = users[b];
      seen = seen_idx + seen_ptr[u];
      n_seen = seen_ptr[u + 1] - seen_ptr[u];
    }
    for (int q = threadIdx.x; q < n; q += TOPN_THREADS) L[q] = cand_masked(L[q], items[q], seen, n_seen, ignore);
    __syncthreads();
    topn_row(L, n, cutoff, items, out_items + (size_t)b * cutoff, out_scores + (size_t)b * cutoff, sm);
  }
}

// the bodies of b200_score_mask_device / b200_score_topn_device and their fp64 twins; `fn` names the entry point in errors
template <typename T>
void score_mask(const char* fn, const int32_t* d_users, int n_users_block, const int32_t* d_urm_ptr, const int32_t* d_urm_idx,
                const unsigned char* d_items_keep, int n_items, T* d_scores, void* stream) {
  B200_REQUIRE(d_scores && n_items > 0 && n_users_block >= 0, "%s: bad argument", fn);
  if (n_users_block == 0) return;
  cudaStream_t st = (cudaStream_t)stream;
  if (d_items_keep) {
    mask_items_kernel<<<div_up((long long)n_users_block * n_items, 256), 256, 0, st>>>(d_items_keep, n_users_block, n_items, d_scores);
    count_launch();
  }
  if (d_users && d_urm_ptr && d_urm_idx) {
    mask_seen_kernel<<<div_up((long long)n_users_block * 32, 256), 256, 0, st>>>(d_users, n_users_block, d_urm_ptr, d_urm_idx, n_items, d_scores);
    count_launch();
  }
  B200_CUDA(cudaGetLastError());
}

template <typename T>
void score_topn(const char* fn, const T* d_scores, int n_rows, int n_items, int cutoff, int32_t* d_items, float* d_item_scores,
                void* stream) {
  B200_REQUIRE(d_scores && d_items && d_item_scores, "%s: NULL argument", fn);
  B200_REQUIRE(cutoff >= 1 && cutoff <= TOPN_MAX, "%s: cutoff must be in [1, %d]", fn, TOPN_MAX);
  if (n_rows == 0) return;
  topn_rows_kernel<<<std::min(n_rows, sm_count() * 8), TOPN_THREADS, 0, (cudaStream_t)stream>>>(d_scores, n_rows, n_items, cutoff,
                                                                                                d_items, d_item_scores);
  B200_CUDA(cudaGetLastError());
  count_launch();
}

}  // namespace score
}  // namespace b200

using namespace b200;
using namespace b200::score;

extern "C" {

int b200_score_spmm_device(const int32_t* d_users, int n_users_block, const int32_t* d_a_ptr, const int32_t* d_a_idx,
                           const float* d_a_val, const int32_t* d_b_ptr, const int32_t* d_b_idx, const float* d_b_val,
                           int n_out_cols, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_a_ptr && d_b_val && d_out, "b200_score_spmm: NULL argument");
    B200_REQUIRE(n_users_block >= 0 && n_out_cols > 0, "b200_score_spmm: bad shape");
    if (n_users_block == 0) return;
    spmm_rows_kernel<<<std::min(n_users_block, sm_count() * 4), 512, 0, (cudaStream_t)stream>>>(
        d_users, n_users_block, d_a_ptr, d_a_idx, d_a_val, d_b_ptr, d_b_idx, d_b_val, n_out_cols, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_transpose_device(const float* d_in, int rows, int cols, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_in && d_out && rows > 0 && cols > 0, "b200_transpose: bad argument");
    transpose_kernel<<<dim3(div_up(cols, 32), std::min(div_up(rows, 32), 65535u)), dim3(32, 8), 0, (cudaStream_t)stream>>>(
        d_in, rows, cols, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_score_mf_device(const int32_t* d_users, int n_users_block, const float* d_user_factors, const float* d_item_factors_T,
                         int n_factors, int n_items, const float* d_user_bias, const float* d_item_bias,
                         const float* d_global_bias, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_user_factors && d_item_factors_T && d_out, "b200_score_mf: NULL argument");
    B200_REQUIRE(n_factors >= 1 && n_items > 0 && n_users_block >= 0, "b200_score_mf: bad shape");
    B200_REQUIRE((d_global_bias == nullptr) == (d_user_bias == nullptr) && (d_user_bias == nullptr) == (d_item_bias == nullptr),
                 "b200_score_mf: biases must be all given or all NULL");
    if (n_users_block == 0) return;
    const size_t smem = (size_t)UT * n_factors * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "b200_score_mf: n_factors=%d too large", n_factors);
    // gridDim.y (UT users per block) is capped at 65 535: larger user arrays take several launches
    const int per_launch = 65535 * UT;
    for (int b0 = 0; b0 < n_users_block; b0 += per_launch) {
      const int nb = std::min(per_launch, n_users_block - b0);
      mf_scores_kernel<<<dim3(div_up(n_items, 256), div_up(nb, UT)), 256, smem, (cudaStream_t)stream>>>(
          d_users + b0, nb, d_user_factors, d_item_factors_T, n_factors, n_items, d_user_bias, d_item_bias, d_global_bias,
          d_out + (size_t)b0 * n_items);
      B200_CUDA(cudaGetLastError());
      count_launch();
    }
  });
}

int b200_score_mask_device(const int32_t* d_users, int n_users_block, const int32_t* d_urm_ptr, const int32_t* d_urm_idx,
                           const unsigned char* d_items_keep, int n_items, float* d_scores, void* stream) {
  return guarded([&] { score_mask("b200_score_mask", d_users, n_users_block, d_urm_ptr, d_urm_idx, d_items_keep, n_items, d_scores, stream); });
}

int b200_score_mask_f64_device(const int32_t* d_users, int n_users_block, const int32_t* d_urm_ptr, const int32_t* d_urm_idx,
                               const unsigned char* d_items_keep, int n_items, double* d_scores, void* stream) {
  return guarded([&] {
    score_mask("b200_score_mask_f64", d_users, n_users_block, d_urm_ptr, d_urm_idx, d_items_keep, n_items, d_scores, stream);
  });
}

int b200_score_topn_device(const float* d_scores, int n_rows, int n_items, int cutoff, int32_t* d_items, float* d_item_scores,
                           void* stream) {
  return guarded([&] { score_topn("b200_score_topn", d_scores, n_rows, n_items, cutoff, d_items, d_item_scores, stream); });
}

int b200_score_topn_f64_device(const double* d_scores, int n_rows, int n_items, int cutoff, int32_t* d_items,
                               float* d_item_scores, void* stream) {
  return guarded([&] { score_topn("b200_score_topn_f64", d_scores, n_rows, n_items, cutoff, d_items, d_item_scores, stream); });
}

int b200_cand_score_sparse_device(const int32_t* d_users, int n_block, const int32_t* d_a_ptr, const int32_t* d_a_idx,
                                  const float* d_a_val, const int32_t* d_b_ptr, const int32_t* d_b_idx, const float* d_b_val,
                                  const int32_t* d_cand_ptr, const int32_t* d_cand_idx, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_a_ptr && d_a_idx && d_a_val && d_b_ptr && d_b_idx && d_b_val && d_cand_ptr && d_cand_idx && d_out,
                 "b200_cand_score_sparse: NULL argument");
    B200_REQUIRE(n_block >= 0, "b200_cand_score_sparse: bad shape");
    if (n_block == 0) return;
    cand_sparse_kernel<<<n_block, CAND_THREADS, 0, (cudaStream_t)stream>>>(d_users, d_a_ptr, d_a_idx, d_a_val, d_b_ptr, d_b_idx,
                                                                            d_b_val, d_cand_ptr, d_cand_idx, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_cand_score_dense_device(const int32_t* d_users, int n_block, const int32_t* d_a_ptr, const int32_t* d_a_idx,
                                 const float* d_a_val, const float* d_B, int n_items, const int32_t* d_cand_ptr,
                                 const int32_t* d_cand_idx, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_a_ptr && d_a_idx && d_a_val && d_B && d_cand_ptr && d_cand_idx && d_out,
                 "b200_cand_score_dense: NULL argument");
    B200_REQUIRE(n_block >= 0 && n_items > 0, "b200_cand_score_dense: bad shape");
    if (n_block == 0) return;
    cand_dense_kernel<<<n_block, CAND_THREADS, 0, (cudaStream_t)stream>>>(d_users, d_a_ptr, d_a_idx, d_a_val, d_B, n_items,
                                                                           d_cand_ptr, d_cand_idx, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_cand_score_mf_device(const int32_t* d_users, int n_block, const float* d_user_factors, const float* d_item_factors,
                              int n_factors, const float* d_user_bias, const float* d_item_bias, const float* d_global_bias,
                              const int32_t* d_cand_ptr, const int32_t* d_cand_idx, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_user_factors && d_item_factors && d_cand_ptr && d_cand_idx && d_out, "b200_cand_score_mf: NULL argument");
    B200_REQUIRE(n_factors >= 1 && n_block >= 0, "b200_cand_score_mf: bad shape");
    B200_REQUIRE((d_global_bias == nullptr) == (d_user_bias == nullptr) && (d_user_bias == nullptr) == (d_item_bias == nullptr),
                 "b200_cand_score_mf: biases must be all given or all NULL");
    const size_t smem = (size_t)n_factors * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "b200_cand_score_mf: n_factors=%d too large", n_factors);
    if (n_block == 0) return;
    cand_mf_kernel<<<n_block, CAND_THREADS, smem, (cudaStream_t)stream>>>(d_users, d_user_factors, d_item_factors, n_factors,
                                                                           d_user_bias, d_item_bias, d_global_bias, d_cand_ptr,
                                                                           d_cand_idx, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_cand_gather_device(int n_block, const float* d_scores, int n_items, const int32_t* d_cand_ptr, const int32_t* d_cand_idx,
                            float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_scores && d_cand_ptr && d_cand_idx && d_out, "b200_cand_gather: NULL argument");
    B200_REQUIRE(n_block >= 0 && n_items > 0, "b200_cand_gather: bad shape");
    if (n_block == 0) return;
    cand_gather_kernel<<<div_up((long long)n_block * 32, 256), 256, 0, (cudaStream_t)stream>>>(n_block, d_scores, n_items, d_cand_ptr,
                                                                                             d_cand_idx, d_out);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_cand_topn_device(const int32_t* d_users, int n_block, const int32_t* d_cand_ptr, const int32_t* d_cand_idx,
                          float* d_cand_scores, const int32_t* d_seen_ptr, const int32_t* d_seen_idx, const unsigned char* d_ignore,
                          int cutoff, int32_t* d_items, float* d_item_scores, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_cand_ptr && d_cand_idx && d_cand_scores && d_items && d_item_scores, "b200_cand_topn: NULL argument");
    B200_REQUIRE((d_seen_ptr == nullptr) == (d_seen_idx == nullptr) && (d_seen_ptr == nullptr || d_users),
                 "b200_cand_topn: the seen-item filter needs d_users, d_seen_ptr and d_seen_idx");
    B200_REQUIRE(cutoff >= 1 && cutoff <= TOPN_MAX, "b200_cand_topn: cutoff must be in [1, %d]", TOPN_MAX);
    B200_REQUIRE(n_block >= 0, "b200_cand_topn: bad shape");
    if (n_block == 0) return;
    cudaStream_t st = (cudaStream_t)stream;
    cand_topn_warp_kernel<<<div_up(n_block, CAND_TOPN_WARPS), CAND_TOPN_WARPS * 32, 0, st>>>(
        d_users, n_block, d_cand_ptr, d_cand_idx, d_cand_scores, d_seen_ptr, d_seen_idx, d_ignore, cutoff, d_items, d_item_scores);
    B200_CUDA(cudaGetLastError());
    cand_topn_cta_kernel<<<std::min(n_block, sm_count() * 4), TOPN_THREADS, 0, st>>>(
        d_users, n_block, d_cand_ptr, d_cand_idx, d_cand_scores, d_seen_ptr, d_seen_idx, d_ignore, cutoff, d_items, d_item_scores);
    B200_CUDA(cudaGetLastError());
    count_launch(2);
  });
}

}  // extern "C"
