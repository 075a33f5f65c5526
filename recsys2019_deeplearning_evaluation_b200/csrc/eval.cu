// Evaluation inner loop fused behind the top-N kernel (SURVEY.md 8(f).1), sm_90a.
//
// Replaces Base/Evaluation/Evaluator.py:305-388 (_compute_metrics_on_recommendation_list) and the per-user functions of
// Base/Evaluation/metrics.py it calls: precision :214, precision_recall_min_denominator :225, recall :237,
// average_precision :65 / _min_denominator :106, rr :146, ndcg :247 (graded relevance = the test rating, 2^r - 1 gains),
// arhr_all_hits :200, HIT_RATE :164, Novelty :615 (its per-item term is -log2(pop/n_interactions)/n_items, :651),
// AveragePopularity :670, and the per-item recommendation counters every global-distribution metric is a function of
// (_Global_Item_Distribution_Counter :289, Coverage_Item_HIT :346, Diversity_MeanInterList :778).
//
// Input: the [n_block, max_cutoff] item table of b200_score_topn_device (entries whose score is not finite are not
// recommendations, BaseRecommender.py:203-207 drops them) and the test URM in CSR on the device.  One warp per user: the
// hit flag / gain of every recommendation is found by a binary search in the user's sorted test row, hits are
// prefix-summed with ballots, then every cutoff (any number, any order) reduces its prefix of the list.  Sums go to fp64
// accumulators with atomics; nothing returns to the host until the evaluation ends.  HBM-bound on the list table (4 B per
// position) and the test rows.  DIVERSITY_SIMILARITY (Diversity_similarity :719, a dense item x item matrix) has a kernel
// of its own below, launched on the same table only when the evaluator was given a diversity object.
#include "common.cuh"

namespace b200 {
namespace eval {

constexpr int WARPS = 4;
constexpr int MAXCUT = 1024;  // list positions per user (b200_score_topn_device's limit)

// The one definition of a user's recommendation list, shared by every kernel here.  A warp walks the table row
// srow / row 32 positions per step (p0 = 0, 32, ...): the lane's entry is a recommendation iff its score is finite
// (BaseRecommender.py:203-207 drops the rest from the first max_cutoff positions), and the recommendations are compacted
// to list positions 0..len-1 in table order, so +inf entries before them and NaN / -inf entries among them take no
// position.  Returns the lane's item (-1 if none) and its list position in `pos`; advances `len` for the whole warp.
__device__ __forceinline__ int list_step(const int* row, const float* srow, int max_cutoff, int p0, int lane, int& len,
                                         int& pos) {
  const int p = p0 + lane;
  int item = -1;
  if (p < max_cutoff && isfinite(srow[p])) item = row[p];
  const unsigned valid_mask = __ballot_sync(0xffffffffu, item >= 0);
  pos = len + __popc(valid_mask & ((1u << lane) - 1u));
  len += __popc(valid_mask);
  return item;
}

__global__ void __launch_bounds__(WARPS * 32) metrics_kernel(
    const int* __restrict__ users, int n_block, const int* __restrict__ rec, const float* __restrict__ rec_score, int max_cutoff,
    const int* __restrict__ t_ptr, const int* __restrict__ t_idx, const float* __restrict__ t_val,
    const int* __restrict__ cutoffs, int n_cut, const double* __restrict__ idcg, const double* __restrict__ item_novelty,
    const double* __restrict__ item_pop_norm, int n_items, double* acc, int* rec_count, int* hit_count) {
  __shared__ float s_gain[WARPS][MAXCUT];          // 2^rating - 1 of a hit, 0 otherwise
  __shared__ unsigned short s_cum[WARPS][MAXCUT];  // hits among positions 0..p
  __shared__ int s_item[WARPS][MAXCUT];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int b = blockIdx.x * WARPS + w;
  if (b >= n_block) return;
  const int u = users[b];
  const int ts = t_ptr[u], te = t_ptr[u + 1];
  const int n_test = te - ts;
  const int* row = rec + (size_t)b * max_cutoff;
  const float* srow = rec_score + (size_t)b * max_cutoff;
  // ---- phase 1: hit / gain per recommendation, running hit count, list length (the list of list_step)
  int carry = 0, len = 0;
  for (int p0 = 0; p0 < max_cutoff; p0 += 32) {
    int q;  // position among the recommendations
    const int item = list_step(row, srow, max_cutoff, p0, lane, len, q);
    int hit = 0;
    float gain = 0.f;
    if (item >= 0) {
      int lo = ts, hi = te;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t_idx[mid] < item) lo = mid + 1; else hi = mid;
      }
      if (lo < te && t_idx[lo] == item) { hit = 1; gain = exp2f(t_val[lo]) - 1.f; }
    }
    const unsigned hit_mask = __ballot_sync(0xffffffffu, hit);
    if (item >= 0) {
      s_item[w][q] = item;
      s_gain[w][q] = gain;
      s_cum[w][q] = (unsigned short)(carry + __popc(hit_mask & (0xffffffffu >> (31 - lane))));
    }
    carry += __popc(hit_mask);
  }
  __syncwarp();
  // ---- phase 2: every cutoff reduces its prefix of the list
  for (int ci = 0; ci < n_cut; ++ci) {
    const int c = cutoffs[ci];
    const int L = min(c, len);  // len(is_relevant[0:cutoff])
    double ap = 0.0, arhr = 0.0, dcg = 0.0, nov = 0.0, pop = 0.0;
    int hits = 0, first = 1 << 30;
    for (int p = lane; p < L; p += 32) {
      const int item = s_item[w][p];
      const float g = s_gain[w][p];
      const int cum = s_cum[w][p];
      const int prev = p ? s_cum[w][p - 1] : 0;
      const int hit = cum - prev;
      if (hit) {
        ++hits;
        first = min(first, p);
        ap += (double)cum / (double)(p + 1);
        arhr += 1.0 / (double)(p + 1);
        dcg += (double)g / log2((double)p + 2.0);
        atomicAdd(hit_count + (size_t)ci * n_items + item, 1);
      }
      nov += item_novelty[item];
      pop += item_pop_norm[item];
      atomicAdd(rec_count + (size_t)ci * n_items + item, 1);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      ap += __shfl_xor_sync(0xffffffffu, ap, off);
      arhr += __shfl_xor_sync(0xffffffffu, arhr, off);
      dcg += __shfl_xor_sync(0xffffffffu, dcg, off);
      nov += __shfl_xor_sync(0xffffffffu, nov, off);
      pop += __shfl_xor_sync(0xffffffffu, pop, off);
      hits += __shfl_xor_sync(0xffffffffu, hits, off);
      first = min(first, __shfl_xor_sync(0xffffffffu, first, off));
    }
    if (lane == 0) {
      double* a = acc + (size_t)ci * B200_EVAL_NACC;
      const double h = (double)hits;
      if (L > 0) {
        atomicAdd(a + B200_EVAL_PRECISION, h / (double)L);
        atomicAdd(a + B200_EVAL_PRECISION_RECALL_MIN_DEN, h / (double)min(n_test, L));
        atomicAdd(a + B200_EVAL_MAP, ap / (double)L);
        atomicAdd(a + B200_EVAL_MAP_MIN_DEN, ap / (double)min(n_test, L));
        atomicAdd(a + B200_EVAL_AVERAGE_POPULARITY, pop / (double)L);
        atomicAdd(a + B200_EVAL_USERS_WITH_RECS, 1.0);
      }
      atomicAdd(a + B200_EVAL_RECALL, h / (double)n_test);
      if (hits) {
        atomicAdd(a + B200_EVAL_MRR, 1.0 / (double)(first + 1));
        atomicAdd(a + B200_EVAL_HIT_RATE, 1.0);
        atomicAdd(a + B200_EVAL_ARHR, arhr);
        const double ideal = idcg[(size_t)u * n_cut + ci];
        if (dcg != 0.0 && ideal != 0.0) atomicAdd(a + B200_EVAL_NDCG, dcg / ideal);
      }
      atomicAdd(a + B200_EVAL_NOVELTY, nov);
      atomicAdd(a + B200_EVAL_N_USERS, 1.0);
    }
  }
}

// ---- intra-list diversity (Diversity_similarity.add_recommendations, metrics.py:733-741)
// S(L) = sum over a <= L-2, b <= L-1, b != a of D[r_a, r_b].  A term (a, b) first appears at list length
// max(a + 2, b + 1), so with e = max(a + 1, b) the terms fall into buckets
//   T_e = sum_{b <= e, b != e-1} D[r_{e-1}, r_b] + sum_{a <= e-2} D[r_a, r_e]      (2e - 1 terms, e >= 1)
// and S(L) = T_1 + ... + T_{L-1} for every L at once.  One CTA per user: warp 0 puts the list in shared memory, the warps
// take the buckets e = 1 .. L_max - 1 in turn, so each term of D is read once ((L_max - 1)^2 reads, one 32-byte sector
// each at worst), and then every cutoff sums its buckets.  Each sum runs in a fixed order (lane-strided, then a shuffle
// tree), so a user's S does not depend on scheduling; across users values meet in fp64 atomics, like metrics_kernel's.
constexpr int DIV_WARPS = 8;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(DIV_WARPS * 32) diversity_kernel(
    const int* __restrict__ rec, const float* __restrict__ rec_score, int max_cutoff, const int* __restrict__ cutoffs, int n_cut,
    const T* __restrict__ D, int n_items, double* acc) {
  __shared__ int s_item[MAXCUT];
  __shared__ double s_bucket[MAXCUT];  // T_e
  __shared__ int s_len;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (w == 0) {
    const int* row = rec + (size_t)blockIdx.x * max_cutoff;
    const float* srow = rec_score + (size_t)blockIdx.x * max_cutoff;
    int len = 0;
    for (int p0 = 0; p0 < max_cutoff; p0 += 32) {
      int q;
      const int item = list_step(row, srow, max_cutoff, p0, lane, len, q);
      if (item >= 0) s_item[q] = item;
    }
    if (lane == 0) s_len = len;
  }
  __syncthreads();
  const int len = s_len;
  int lmax = 0;
  for (int ci = 0; ci < n_cut; ++ci) lmax = max(lmax, min(cutoffs[ci], len));
  for (int e = 1 + w; e < lmax; e += DIV_WARPS) {
    const T* drow = D + (size_t)s_item[e - 1] * n_items;  // row r_{e-1}
    const int re = s_item[e];                              // column r_e
    double t = 0.0;
#pragma unroll 4
    for (int b = lane; b <= e; b += 32) t += b == e - 1 ? 0.0 : (double)drow[s_item[b]];
#pragma unroll 4
    for (int a = lane; a <= e - 2; a += 32) t += (double)D[(size_t)s_item[a] * n_items + re];
    t = warp_sum(t);
    if (lane == 0) s_bucket[e] = t;
  }
  __syncthreads();
  for (int ci = w; ci < n_cut; ci += DIV_WARPS) {
    const int L = min(cutoffs[ci], len);
    double s = 0.0;
    for (int e = 1 + lane; e < L; e += 32) s += s_bucket[e];
    s = warp_sum(s);
    if (lane == 0) {
      double* a = acc + (size_t)ci * B200_EVAL_NACC;
      if (L < 2) atomicAdd(a + B200_EVAL_SHORT_LISTS, 1.0);
      else atomicAdd(a + B200_EVAL_DIVERSITY_SIMILARITY, s / ((double)L * (double)(L - 1)));
    }
  }
}

}  // namespace eval
}  // namespace b200

using namespace b200;

extern "C" {

int b200_eval_accumulate_device(const int32_t* d_users, int n_block, const int32_t* d_rec_items, const float* d_rec_scores,
                                int max_cutoff, const int32_t* d_test_ptr, const int32_t* d_test_idx, const float* d_test_val,
                                const int32_t* d_cutoffs, int n_cutoffs, const double* d_idcg, const double* d_item_novelty,
                                const double* d_item_pop_norm, int n_items, double* d_acc, int32_t* d_rec_count,
                                int32_t* d_hit_count, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_users && d_rec_items && d_rec_scores && d_test_ptr && d_test_idx && d_test_val && d_cutoffs && d_idcg &&
                     d_item_novelty && d_item_pop_norm && d_acc && d_rec_count && d_hit_count,
                 "b200_eval_accumulate: NULL argument");
    B200_REQUIRE(max_cutoff >= 1 && max_cutoff <= eval::MAXCUT, "b200_eval_accumulate: max_cutoff must be in [1, %d]", eval::MAXCUT);
    B200_REQUIRE(n_cutoffs >= 1 && n_items > 0 && n_block >= 0, "b200_eval_accumulate: bad shape");
    if (n_block == 0) return;
    eval::metrics_kernel<<<div_up(n_block, eval::WARPS), eval::WARPS * 32, 0, (cudaStream_t)stream>>>(
        d_users, n_block, d_rec_items, d_rec_scores, max_cutoff, d_test_ptr, d_test_idx, d_test_val, d_cutoffs, n_cutoffs, d_idcg,
        d_item_novelty, d_item_pop_norm, n_items, d_acc, d_rec_count, d_hit_count);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_eval_diversity_device(const int32_t* d_rec_items, const float* d_rec_scores, int n_block, int max_cutoff,
                               const int32_t* d_cutoffs, int n_cutoffs, const void* d_div, int div_fp64, int n_items,
                               double* d_acc, void* stream) {
  return guarded([&] {
    B200_REQUIRE(d_rec_items && d_rec_scores && d_cutoffs && d_div && d_acc, "b200_eval_diversity: NULL argument");
    B200_REQUIRE(max_cutoff >= 1 && max_cutoff <= eval::MAXCUT, "b200_eval_diversity: max_cutoff must be in [1, %d]", eval::MAXCUT);
    B200_REQUIRE(n_cutoffs >= 1 && n_items > 0 && n_block >= 0, "b200_eval_diversity: bad shape");
    if (n_block == 0) return;
    const cudaStream_t s = (cudaStream_t)stream;
    if (div_fp64)
      eval::diversity_kernel<double><<<n_block, eval::DIV_WARPS * 32, 0, s>>>(
          d_rec_items, d_rec_scores, max_cutoff, d_cutoffs, n_cutoffs, static_cast<const double*>(d_div), n_items, d_acc);
    else
      eval::diversity_kernel<float><<<n_block, eval::DIV_WARPS * 32, 0, s>>>(
          d_rec_items, d_rec_scores, max_cutoff, d_cutoffs, n_cutoffs, static_cast<const float*>(d_div), n_items, d_acc);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

}  // extern "C"
