// K3: SLIM-BPR epochs on a dense (optionally symmetric) item-item matrix S, sm_90a.
//
// Replaces SLIM_BPR/Cython/SLIM_BPR_Cython_Epoch.pyx: epochIteration_Cython :211-335, sampleBPR_Cython :436-480,
// adaptive_gradient :395-433 (per-ITEM scalar state shared by the positive and negative roles), symmetric storage
// Triangular_Matrix :1272-1330, get_S :340-388 (diagonal zeroed).  S is dense fp32 in HBM (C2: 55 MB, L2-resident).
// The tree-sparse training mode (train_with_sparse_weights, Sparse_Matrix_Tree_CSR :579-1031) keeps its SEMANTICS on the
// same dense array: a byte map records which cells the reference's row trees would hold, and the periodic
// rebalance_tree(TopK) :782-802 / the in-place selection of get_scipy_csr(TopK) :762-763 is slim_tree_prune_kernel.
//
// Two execution modes (DESIGN.md "K3"):
//   * sequential (the reference's semantics exactly): the recursion is batch-1 and every sample reads cells the
//     previous one may have written, so ONE CTA walks the replayed sample stream in order; the 2*len_u cell reads,
//     the x_uij reduction and the 2*len_u updates of a sample are spread over the CTA's threads.
//   * hogwild: all SMs, one warp per sample, float atomics on S (Hogwild races), Philox or replayed stream.
// Roofline: HBM/L2, 4*len_u*4 bytes per sample for S (two row gathers read + written) + 4*len_u for the profile.
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace b200 {
namespace slim {

enum SgdMode { SGD = 0, ADAGRAD = 1, RMSPROP = 2, ADAM = 3 };

struct Params {
  int n_users, n_items, symmetric, sgd_mode;
  float lr, li_reg, lj_reg, gamma, beta1, beta2;
  double b1_pow, b2_pow;
  const int* __restrict__ indptr;
  const int* __restrict__ indices;
  float* S;                // n_items x n_items row-major; symmetric mode uses the lower triangle (row >= col)
  float *c, *m1, *m2;      // per-item adaptive state
  const int* su; const int* si; const int* sj;
  long long n_samples;
  double* pow_out;
  unsigned char* exists;   // tree mode: 1 where the reference's row tree holds a cell (add_value creates it, pyx:617-680)
  long long first;         // first sample of this launch (tree mode runs an epoch as segments between two prunings)
  int chain_pow;           // continue the Adam powers from pow_out (segment > 0) instead of b1_pow / b2_pow
  int prof;                // B200REC_SLIM_PROF=1: thread 0 times the phases of the sequential kernel (development hook)
};

__device__ __forceinline__ size_t cell(const Params& p, int a, int b) {
  if (p.symmetric && b > a) { const int t = a; a = b; b = t; }  // pyx:1287-1302, 1309-1330
  return (size_t)a * p.n_items + b;
}

__device__ __forceinline__ float adapt_item(const Params& p, float g, int item, float inv1, float inv2) {  // pyx:395-433
  if (p.sgd_mode == ADAGRAD) {
    const float cc = p.c[item] + g * g;
    p.c[item] = cc;
    return g / (sqrtf(cc) + 1e-8f);
  } else if (p.sgd_mode == RMSPROP) {
    const float cc = p.c[item] * p.gamma + (1.f - p.gamma) * g * g;
    p.c[item] = cc;
    return g / (sqrtf(cc) + 1e-8f);
  } else if (p.sgd_mode == ADAM) {
    const float a = p.m1[item] * p.beta1 + (1.f - p.beta1) * g;
    const float b = p.m2[item] * p.beta2 + (1.f - p.beta2) * g * g;
    p.m1[item] = a;
    p.m2[item] = b;
    return (a * inv1) / (sqrtf(b * inv2) + 1e-8f);
  }
  return g;
}

constexpr int SEQ_THREADS = 512;
constexpr int SEQ_WARPS = SEQ_THREADS / 32;

#define SLIM_MARK(k) do { if (p.prof && tid == 0) { const long long t_ = clock64(); prof[k] += (unsigned long long)(t_ - tprev); tprev = t_; } } while (0)
// one CTA, samples strictly in order (pyx:231-312).  The next sample's (u, i, j), its profile bounds and this thread's
// profile entry are fetched while the current sample runs, and thread 0 requests the adaptive state of i and j before the
// reduction: what is left on the critical path of a sample is one trip for the S cells, the reduction, the gradient, and the
// update of cells that are in L1 by then.
__global__ void __launch_bounds__(SEQ_THREADS) slim_sequential_kernel(const Params p) {
  __shared__ float red[SEQ_WARPS];
  __shared__ float s_gi, s_gj;
  __shared__ unsigned long long prof[6];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double b1p = p.chain_pow ? p.pow_out[0] : p.b1_pow, b2p = p.chain_pow ? p.pow_out[1] : p.b2_pow;
  long long tprev = 0;
  if (tid < 6) prof[tid] = 0ull;
  __syncthreads();  // pow_out is rewritten at the end
  const long long last = p.first + p.n_samples;
  // sample n in (u, i, j, s, e, sn0); sample n + 1 in (nu, ni, nj)
  int u = 0, i = 0, j = 0, s = 0, e = 0, sn0 = -1, nu = 0, ni = 0, nj = 0;
  if (p.n_samples > 0) {
    u = p.su[p.first]; i = p.si[p.first]; j = p.sj[p.first];
    s = p.indptr[u]; e = p.indptr[u + 1];
    if (s + tid < e) sn0 = p.indices[s + tid];
  }
  if (p.n_samples > 1) { nu = p.su[p.first + 1]; ni = p.si[p.first + 1]; nj = p.sj[p.first + 1]; }
  if (p.prof && tid == 0) tprev = clock64();
  for (long long n = p.first; n < last; ++n) {
    int nnu = 0, nni = 0, nnj = 0;
    if (n + 2 < last) { nnu = p.su[n + 2]; nni = p.si[n + 2]; nnj = p.sj[n + 2]; }
    const int ns = p.indptr[nu], ne = p.indptr[nu + 1];  // nu arrived an iteration ago (user 0 past the end: harmless)
    // thread 0: the adaptive state of i and j, in flight during the gather (pyx:395-433 reads it after the gradient)
    float st_i0 = 0.f, st_i1 = 0.f, st_j0 = 0.f, st_j1 = 0.f;
    if (tid == 0) {
      if (p.sgd_mode == ADAGRAD || p.sgd_mode == RMSPROP) { st_i0 = p.c[i]; st_j0 = p.c[j]; }
      else if (p.sgd_mode == ADAM) { st_i0 = p.m1[i]; st_i1 = p.m2[i]; st_j0 = p.m1[j]; st_j1 = p.m2[j]; }
    }
    float x = 0.f;
    if (sn0 >= 0) x = p.S[cell(p, i, sn0)] - p.S[cell(p, j, sn0)];  // pyx:242-255
    for (int k = s + tid + SEQ_THREADS; k < e; k += SEQ_THREADS) {
      const int sn = p.indices[k];
      x += p.S[cell(p, i, sn)] - p.S[cell(p, j, sn)];
    }
    int nsn0 = -1;
    if (ns + tid < ne) nsn0 = p.indices[ns + tid];  // the next sample's profile entry of this thread
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    if (lane == 0) red[warp] = x;
    SLIM_MARK(0);
    __syncthreads();
    SLIM_MARK(1);
    if (warp == 0) {
      float t = lane < SEQ_WARPS ? red[lane] : 0.f;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
      if (lane == 0) {
        const float g = 1.f / (1.f + expf(t));  // pyx:258
        const float inv1 = (float)(1.0 / (1.0 - b1p)), inv2 = (float)(1.0 / (1.0 - b2p));
        float gi = g, gj = g;  // i first, then j (pyx:262-263); i != j always (j is not in the profile, i is)
        if (p.sgd_mode == ADAGRAD) {
          st_i0 += g * g; gi = g / (sqrtf(st_i0) + 1e-8f); p.c[i] = st_i0;
          st_j0 += g * g; gj = g / (sqrtf(st_j0) + 1e-8f); p.c[j] = st_j0;
        } else if (p.sgd_mode == RMSPROP) {
          st_i0 = st_i0 * p.gamma + (1.f - p.gamma) * g * g; gi = g / (sqrtf(st_i0) + 1e-8f); p.c[i] = st_i0;
          st_j0 = st_j0 * p.gamma + (1.f - p.gamma) * g * g; gj = g / (sqrtf(st_j0) + 1e-8f); p.c[j] = st_j0;
        } else if (p.sgd_mode == ADAM) {
          st_i0 = st_i0 * p.beta1 + (1.f - p.beta1) * g; st_i1 = st_i1 * p.beta2 + (1.f - p.beta2) * g * g;
          gi = (st_i0 * inv1) / (sqrtf(st_i1 * inv2) + 1e-8f); p.m1[i] = st_i0; p.m2[i] = st_i1;
          st_j0 = st_j0 * p.beta1 + (1.f - p.beta1) * g; st_j1 = st_j1 * p.beta2 + (1.f - p.beta2) * g * g;
          gj = (st_j0 * inv1) / (sqrtf(st_j1 * inv2) + 1e-8f); p.m1[j] = st_j0; p.m2[j] = st_j1;
        }
        s_gi = gi; s_gj = gj;
      }
    }
    SLIM_MARK(2);
    __syncthreads();
    SLIM_MARK(3);
    const float gi = s_gi, gj = s_gj;
    // pyx:266-304.  Within one sample the cells (i, s) are distinct from each other and from the cells (j, s')
    // except in symmetric mode where (i, j) and (j, i) coincide when both i and j are in the profile -- j never is
    // (it is a sampled negative), so the cell sets are disjoint and the order inside the sample is free.
    for (int k = s + tid; k < e; k += SEQ_THREADS) {
      const int sn = k == s + tid ? sn0 : p.indices[k];
      if (sn != i) {
        const size_t c = cell(p, i, sn); const float v = p.S[c]; p.S[c] = v + p.lr * (gi - p.li_reg * v);
        if (p.exists) p.exists[c] = 1;
      }
      if (sn != j) {
        const size_t c = cell(p, j, sn); const float v = p.S[c]; p.S[c] = v - p.lr * (gj - p.lj_reg * v);
        if (p.exists) p.exists[c] = 1;
      }
    }
    if (p.sgd_mode == ADAM) { b1p *= (double)p.beta1; b2p *= (double)p.beta2; }  // per sample, pyx:309-312
    u = nu; i = ni; j = nj; s = ns; e = ne; sn0 = nsn0;
    nu = nnu; ni = nni; nj = nnj;
    SLIM_MARK(4);
    __syncthreads();
    SLIM_MARK(5);
  }
  if (tid == 0) {
    p.pow_out[0] = b1p; p.pow_out[1] = b2p;
    if (p.prof && p.n_samples > 0)
      printf("slim sequential phase cycles per sample: gather=%llu bar1=%llu gradient=%llu bar2=%llu update=%llu bar3=%llu\n",
             prof[0] / p.n_samples, prof[1] / p.n_samples, prof[2] / p.n_samples, prof[3] / p.n_samples, prof[4] / p.n_samples,
             prof[5] / p.n_samples);
  }
}

// all SMs, one warp per sample, no ordering between samples
__global__ void __launch_bounds__(256) slim_hogwild_kernel(const Params p) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long n = warp; n < p.n_samples; n += n_warps) {
    const int u = p.su[n], i = p.si[n], j = p.sj[n];
    const int s = p.indptr[u], e = p.indptr[u + 1];
    float x = 0.f;
    for (int k = s + lane; k < e; k += 32) {
      const int sn = p.indices[k];
      x += p.S[cell(p, i, sn)] - p.S[cell(p, j, sn)];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    const float g = 1.f / (1.f + expf(x));
    float gi = g, gj = g;
    if (p.sgd_mode != SGD) {
      float inv1 = 1.f, inv2 = 1.f;
      if (p.sgd_mode == ADAM) {
        inv1 = (float)(1.0 / (1.0 - p.b1_pow * pow((double)p.beta1, (double)n)));
        inv2 = (float)(1.0 / (1.0 - p.b2_pow * pow((double)p.beta2, (double)n)));
      }
      if (lane == 0) { gi = adapt_item(p, g, i, inv1, inv2); gj = adapt_item(p, g, j, inv1, inv2); }
      gi = __shfl_sync(0xffffffffu, gi, 0);
      gj = __shfl_sync(0xffffffffu, gj, 0);
    }
    for (int k = s + lane; k < e; k += 32) {
      const int sn = p.indices[k];
      if (sn != i) { const size_t c = cell(p, i, sn); atomicAdd(p.S + c, p.lr * (gi - p.li_reg * p.S[c])); }
      if (sn != j) { const size_t c = cell(p, j, sn); atomicAdd(p.S + c, -p.lr * (gj - p.lj_reg * p.S[c])); }
    }
  }
}

// ---- column-sharded S (SURVEY.md 8(e) K3): this rank holds S[:, lo:hi) as an [n_items, width] slab.  Every rank draws the
// same samples (counter-based Philox: same seed, epoch and sample index); a step handles a batch of them against the frozen
// S: each rank sums the cells of its own columns into a partial x_uij per sample, the ranks' partials are added by ONE
// all-reduce of a [batch] vector, and every rank then updates the cells it owns.  batch = 1 is the reference's recursion
// (pyx:231-312) exactly; larger batches trade staleness inside the batch for fewer exchanges.
struct ShardParams {
  Params p;
  int lo, hi, width;
  long long first;  // index of the batch's first sample within the epoch
  int n_batch;
};

__global__ void __launch_bounds__(256) slim_shard_partial_kernel(const ShardParams sp, float* __restrict__ x_out) {
  const Params& p = sp.p;
  const int lane = threadIdx.x & 31;
  const int warp = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int n_warps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int n = warp; n < sp.n_batch; n += n_warps) {
    const long long g = sp.first + n;
    const int u = p.su[g], i = p.si[g], j = p.sj[g];
    const int s = p.indptr[u], e = p.indptr[u + 1];
    const float* Si = p.S + (size_t)i * sp.width - sp.lo;
    const float* Sj = p.S + (size_t)j * sp.width - sp.lo;
    float x = 0.f;
    for (int k = s + lane; k < e; k += 32) {
      const int sn = p.indices[k];
      if (sn >= sp.lo && sn < sp.hi) x += Si[sn] - Sj[sn];  // pyx:242-255, this rank's columns
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    if (lane == 0) x_out[n] = x;
  }
}

// the adaptive scale of one gradient from the item's state AS OF THE START OF THE BATCH plus this sample's own contribution
// (pyx:395-433 without the store); with one sample per batch this is the reference's value exactly
__device__ __forceinline__ float adapt_item_frozen(const Params& p, float g, int item, float inv1, float inv2) {
  if (p.sgd_mode == ADAGRAD) return g / (sqrtf(p.c[item] + g * g) + 1e-8f);
  if (p.sgd_mode == RMSPROP) return g / (sqrtf(p.c[item] * p.gamma + (1.f - p.gamma) * g * g) + 1e-8f);
  if (p.sgd_mode == ADAM) {
    const float a = p.m1[item] * p.beta1 + (1.f - p.beta1) * g;
    const float b = p.m2[item] * p.beta2 + (1.f - p.beta2) * g * g;
    return (a * inv1) / (sqrtf(b * inv2) + 1e-8f);
  }
  return g;
}

__device__ __forceinline__ void ema_atomic(float* addr, float decay, float add) {  // *addr = *addr * decay + add, atomically
  int old = __float_as_int(*addr), assumed;
  do {
    assumed = old;
    old = atomicCAS(reinterpret_cast<int*>(addr), assumed, __float_as_int(__int_as_float(assumed) * decay + add));
  } while (assumed != old);
}

__global__ void __launch_bounds__(256) slim_shard_apply_kernel(const ShardParams sp, const float* __restrict__ x_sum) {
  const Params& p = sp.p;
  const int lane = threadIdx.x & 31;
  const int warp = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int n_warps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int n = warp; n < sp.n_batch; n += n_warps) {
    const long long g = sp.first + n;
    const int u = p.su[g], i = p.si[g], j = p.sj[g];
    const int s = p.indptr[u], e = p.indptr[u + 1];
    const float gr = 1.f / (1.f + expf(x_sum[n]));  // pyx:258
    float gi = gr, gj = gr;
    if (p.sgd_mode != SGD) {
      float inv1 = 1.f, inv2 = 1.f;
      if (p.sgd_mode == ADAM) {  // the powers advance once per sample (pyx:309-312)
        inv1 = (float)(1.0 / (1.0 - p.b1_pow * pow((double)p.beta1, (double)g)));
        inv2 = (float)(1.0 / (1.0 - p.b2_pow * pow((double)p.beta2, (double)g)));
      }
      // the per-item state is replicated and frozen while a batch is applied: every rank derives the same scales
      if (lane == 0) { gi = adapt_item_frozen(p, gr, i, inv1, inv2); gj = adapt_item_frozen(p, gr, j, inv1, inv2); }
      gi = __shfl_sync(0xffffffffu, gi, 0);
      gj = __shfl_sync(0xffffffffu, gj, 0);
    }
    float* Si = p.S + (size_t)i * sp.width - sp.lo;
    float* Sj = p.S + (size_t)j * sp.width - sp.lo;
    for (int k = s + lane; k < e; k += 32) {
      const int sn = p.indices[k];
      if (sn < sp.lo || sn >= sp.hi) continue;
      if (sn != i) atomicAdd(Si + sn, p.lr * (gi - p.li_reg * Si[sn]));   // pyx:266-283
      if (sn != j) atomicAdd(Sj + sn, -p.lr * (gj - p.lj_reg * Sj[sn]));  // pyx:285-304
    }
  }
}

// after the batch's cells are updated: the batch's gradients enter the per-item state (i then j per sample, pyx:262-263;
// the order BETWEEN the samples of a batch is free: a sum for adagrad, an atomic read-modify-write per hit for the averages)
__global__ void slim_shard_state_kernel(const ShardParams sp, const float* __restrict__ x_sum) {
  const Params& p = sp.p;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= sp.n_batch) return;
  const long long g = sp.first + n;
  const float gr = 1.f / (1.f + expf(x_sum[n]));
  const int items[2] = {p.si[g], p.sj[g]};
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    const int it = items[t];
    if (p.sgd_mode == ADAGRAD) atomicAdd(p.c + it, gr * gr);
    else if (p.sgd_mode == RMSPROP) ema_atomic(p.c + it, p.gamma, (1.f - p.gamma) * gr * gr);
    else if (p.sgd_mode == ADAM) { ema_atomic(p.m1 + it, p.beta1, (1.f - p.beta1) * gr); ema_atomic(p.m2 + it, p.beta2, (1.f - p.beta2) * gr * gr); }
  }
}

// ---- tree mode: rebalance_tree(TopK) pyx:782-802 and the in-place selection inside get_scipy_csr(TopK) pyx:762-763, both
// through topK_selection_from_list pyx:954-1031.  A row whose tree holds at least K cells keeps the K largest by value; the
// reference sorts the column-ordered list with a stable qsort on the value, so among equal values the HIGHER columns
// survive: key = (value bits << 32) | column, keep the K largest keys.  Cells that are dropped cease to exist and read as 0.
// One CTA per row, 11-bit radix select over the 64-bit keys (the row is L2-resident across the six passes).
__device__ __forceinline__ unsigned tree_orderable(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__global__ void __launch_bounds__(256) slim_tree_prune_kernel(float* S, unsigned char* exists, int n, int K, int touch_diagonal) {
  typedef unsigned long long u64;
  constexpr int BINS = 2048;
  __shared__ int hist[BINS];
  __shared__ int s_digit, s_need, s_m;
  const int tid = threadIdx.x;
  for (int row = blockIdx.x; row < n; row += gridDim.x) {
    float* Sr = S + (size_t)row * n;
    unsigned char* Er = exists + (size_t)row * n;
    if (tid == 0) {
      s_m = 0;
      if (touch_diagonal) { Sr[row] = 0.f; Er[row] = 1; }  // get_S: add_value(index, index, -get_value(index, index)), pyx:349-350
    }
    __syncthreads();
    int m = 0;
    for (int c = tid; c < n; c += 256) m += Er[c] != 0;
    m = __reduce_add_sync(0xffffffffu, m);
    if ((tid & 31) == 0 && m) atomicAdd(&s_m, m);
    __syncthreads();
    m = s_m;
    __syncthreads();
    if (K <= 0 || m <= K) continue;  // fewer than K cells: the list is returned as it is (pyx:977-978); exactly K: all stay
    u64 prefix = 0, mask = 0;
    int need = K;
    for (int shift = 53; ; shift -= 11) {
      const int sh = max(shift, 0);
      const int nb = shift >= 0 ? 11 : 11 + shift;
      for (int i = tid; i < BINS; i += 256) hist[i] = 0;
      __syncthreads();
      for (int c = tid; c < n; c += 256) {
        if (Er[c]) {
          const u64 key = (((u64)tree_orderable(Sr[c])) << 32) | (u64)(unsigned)c;
          if ((key & mask) == prefix) atomicAdd(&hist[(int)((key >> sh) & ((1u << nb) - 1))], 1);
        }
      }
      __syncthreads();
      if (tid == 0) {  // the need-th largest digit
        int cum = 0;
        for (int b = (1 << nb) - 1; b >= 0; --b) {
          const int cnt = hist[b];
          if (cum + cnt >= need) { s_digit = b; s_need = need - cum; break; }
          cum += cnt;
        }
      }
      __syncthreads();
      prefix |= ((u64)s_digit) << sh;
      mask |= ((u64)((1u << nb) - 1)) << sh;
      need = s_need;
      __syncthreads();
      if (shift <= 0) break;
    }
    for (int c = tid; c < n; c += 256) {
      if (Er[c]) {
        const u64 key = (((u64)tree_orderable(Sr[c])) << 32) | (u64)(unsigned)c;
        if (key < prefix) { Sr[c] = 0.f; Er[c] = 0; }
      }
    }
    __syncthreads();
  }
}

// expands the stored matrix into the full n x n view get_S returns before its top-K (diagonal zeroed, pyx:345-355;
// symmetric mode mirrors the lower triangle, pyx:1363-1372)
__global__ void slim_full_kernel(const float* __restrict__ S, int n, int symmetric, float* out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)n * n) return;
  const int r = (int)(g / n), c = (int)(g % n);
  float v;
  if (r == c) v = 0.f;
  else if (symmetric && c > r) v = S[(size_t)c * n + r];
  else v = S[g];
  out[g] = v;
}

// device Philox sampler (same acceptance rules as sampleBPR_Cython, pyx:436-480)
__device__ __forceinline__ void philox_round(unsigned& c0, unsigned& c1, unsigned& c2, unsigned& c3, unsigned k0, unsigned k1) {
  const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
  const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
  c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
}
__device__ __forceinline__ uint4 philox(unsigned long long idx, unsigned blk, unsigned seed, unsigned epoch) {
  unsigned c0 = (unsigned)idx, c1 = (unsigned)(idx >> 32), c2 = blk, c3 = 0x243F6A88u;
  unsigned k0 = seed, k1 = epoch;
#pragma unroll
  for (int r = 0; r < 10; ++r) { philox_round(c0, c1, c2, c3, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  return make_uint4(c0, c1, c2, c3);
}

__global__ void slim_sample_kernel(const int* __restrict__ indptr, const int* __restrict__ indices, int n_users, int n_items,
                                   long long n_samples, unsigned seed, unsigned epoch, int* su, int* si, int* sj) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_samples) return;
  unsigned blk = 0;
  uint4 cur = philox((unsigned long long)g, blk++, seed, epoch);
  int pos = 0;
  auto next = [&]() {
    if (pos == 4) { cur = philox((unsigned long long)g, blk++, seed, epoch); pos = 0; }
    const unsigned v = pos == 0 ? cur.x : (pos == 1 ? cur.y : (pos == 2 ? cur.z : cur.w));
    ++pos;
    return v;
  };
  int u, s, n;
  do {
    u = (int)(next() % (unsigned)n_users);
    s = indptr[u];
    n = indptr[u + 1] - s;
  } while (n == 0 || n == n_items);
  const int item = indices[s + (int)(next() % (unsigned)n)];
  int neg;
  while (true) {
    neg = (int)(next() % (unsigned)n_items);
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (indices[s + mid] < neg) lo = mid + 1; else hi = mid; }
    if (lo == n || indices[s + lo] != neg) break;
  }
  su[g] = u; si[g] = item; sj[g] = neg;
}

using GlibcRand = GlibcRandHost;  // common.cuh

}  // namespace slim
}  // namespace b200

using namespace b200;
using namespace b200::slim;

struct b200_slim_s {
  Params p{};
  int sampler = 0, hogwild = 0;
  unsigned seed = 1, epoch = 0;
  GlibcRand rng;
  std::vector<int> h_indptr, h_indices, hs_u, hs_i, hs_j;
  DevBuf<int> d_indptr, d_indices, su, si, sj;
  DevBuf<float> S, c, m1, m2;
  DevBuf<double> pow_out;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool timed = false;
  int shard_lo = 0, shard_hi = 0;  // column-sharded handle (b200_slim_create_sharded): S is [n_items, shard_hi - shard_lo]
  long long drawn_epoch = -1;      // the epoch whose sample stream is in su / si / sj
  DevBuf<unsigned char> exists;    // tree mode (b200_slim_enable_tree)
  bool tree = false;
  int tree_topk = 0;
};

extern "C" {

int b200_slim_create(b200_slim_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                     const int32_t* h_indices, float learning_rate, float li_reg, float lj_reg, int symmetric, int sgd_mode,
                     float gamma, float beta_1, float beta_2, int has_seed, uint32_t random_seed, int sampler, int hogwild) {
  if (out) *out = nullptr;
  b200_slim_s* h = nullptr;
  int rc = guarded([&] {
    B200_REQUIRE(out && h_indptr && (nnz == 0 || h_indices), "b200_slim_create: NULL argument");
    B200_REQUIRE(n_users > 0 && n_items > 0 && nnz >= 0 && nnz < (1ll << 31) - 1, "b200_slim_create: bad shape");
    B200_REQUIRE(sgd_mode >= SGD && sgd_mode <= ADAM, "b200_slim_create: unknown sgd_mode %d", sgd_mode);
    B200_REQUIRE((double)n_items * (double)n_items * 4.0 < 1.6e11, "b200_slim_create: dense S does not fit one GPU");
    h = new b200_slim_s();
    Params& p = h->p;
    p.n_users = (int)n_users; p.n_items = (int)n_items; p.symmetric = symmetric != 0; p.sgd_mode = sgd_mode;
    p.lr = learning_rate; p.li_reg = li_reg; p.lj_reg = lj_reg; p.gamma = gamma; p.beta1 = beta_1; p.beta2 = beta_2;
    p.b1_pow = beta_1; p.b2_pow = beta_2;  // pyx:157-158
    h->sampler = sampler; h->hogwild = hogwild != 0;
    h->seed = has_seed ? random_seed : 1u;
    h->rng.seed(h->seed);
    h->h_indptr.assign(h_indptr, h_indptr + n_users + 1);
    h->h_indices.assign(h_indices, h_indices + nnz);
    h->d_indptr.alloc((size_t)n_users + 1);
    h->d_indices.alloc((size_t)std::max<int64_t>(nnz, 1));
    B200_CUDA(cudaMemcpy(h->d_indptr.get(), h_indptr, sizeof(int) * ((size_t)n_users + 1), cudaMemcpyHostToDevice));
    if (nnz) B200_CUDA(cudaMemcpy(h->d_indices.get(), h_indices, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice));
    p.indptr = h->d_indptr.get(); p.indices = h->d_indices.get();
    const size_t cells = (size_t)n_items * (size_t)n_items;
    h->S.alloc(cells);
    B200_CUDA(cudaMemset(h->S.get(), 0, cells * sizeof(float)));  // S starts at zero (pyx:122-125)
    p.S = h->S.get();
    if (sgd_mode == ADAGRAD || sgd_mode == RMSPROP) {
      h->c.alloc((size_t)n_items); B200_CUDA(cudaMemset(h->c.get(), 0, sizeof(float) * (size_t)n_items)); p.c = h->c.get();
    } else if (sgd_mode == ADAM) {
      h->m1.alloc((size_t)n_items); h->m2.alloc((size_t)n_items);
      B200_CUDA(cudaMemset(h->m1.get(), 0, sizeof(float) * (size_t)n_items));
      B200_CUDA(cudaMemset(h->m2.get(), 0, sizeof(float) * (size_t)n_items));
      p.m1 = h->m1.get(); p.m2 = h->m2.get();
    }
    h->su.alloc((size_t)n_users); h->si.alloc((size_t)n_users); h->sj.alloc((size_t)n_users);
    p.su = h->su.get(); p.si = h->si.get(); p.sj = h->sj.get();
    h->pow_out.alloc(2);
    p.pow_out = h->pow_out.get();
    B200_CUDA(cudaEventCreate(&h->ev0));
    B200_CUDA(cudaEventCreate(&h->ev1));
    *out = h;
  });
  if (rc != B200_OK && h) delete h;
  return rc;
}

int b200_slim_create_sharded(b200_slim_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                             const int32_t* h_indices, float learning_rate, float li_reg, float lj_reg, int sgd_mode, float gamma,
                             float beta_1, float beta_2, uint32_t random_seed, int col_lo, int col_hi) {
  if (out) *out = nullptr;
  b200_slim_s* h = nullptr;
  int rc = guarded([&] {
    B200_REQUIRE(out && h_indptr && (nnz == 0 || h_indices), "b200_slim_create_sharded: NULL argument");
    B200_REQUIRE(n_users > 0 && n_items > 0 && nnz >= 0 && nnz < (1ll << 31) - 1, "b200_slim_create_sharded: bad shape");
    B200_REQUIRE(sgd_mode >= SGD && sgd_mode <= ADAM, "b200_slim_create_sharded: unknown sgd_mode %d", sgd_mode);
    B200_REQUIRE(0 <= col_lo && col_lo < col_hi && col_hi <= n_items, "b200_slim_create_sharded: bad column range [%d,%d)", col_lo, col_hi);
    h = new b200_slim_s();
    Params& p = h->p;
    p.n_users = (int)n_users; p.n_items = (int)n_items; p.symmetric = 0; p.sgd_mode = sgd_mode;
    p.lr = learning_rate; p.li_reg = li_reg; p.lj_reg = lj_reg; p.gamma = gamma; p.beta1 = beta_1; p.beta2 = beta_2;
    p.b1_pow = beta_1; p.b2_pow = beta_2;
    h->sampler = 1; h->hogwild = 1;
    h->seed = random_seed;
    h->shard_lo = col_lo; h->shard_hi = col_hi;
    h->d_indptr.alloc((size_t)n_users + 1);
    h->d_indices.alloc((size_t)std::max<int64_t>(nnz, 1));
    B200_CUDA(cudaMemcpy(h->d_indptr.get(), h_indptr, sizeof(int) * ((size_t)n_users + 1), cudaMemcpyHostToDevice));
    if (nnz) B200_CUDA(cudaMemcpy(h->d_indices.get(), h_indices, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice));
    p.indptr = h->d_indptr.get(); p.indices = h->d_indices.get();
    const size_t cells = (size_t)n_items * (size_t)(col_hi - col_lo);
    h->S.alloc(cells);
    B200_CUDA(cudaMemset(h->S.get(), 0, cells * sizeof(float)));
    p.S = h->S.get();
    if (sgd_mode == ADAGRAD || sgd_mode == RMSPROP) {
      h->c.alloc((size_t)n_items); B200_CUDA(cudaMemset(h->c.get(), 0, sizeof(float) * (size_t)n_items)); p.c = h->c.get();
    } else if (sgd_mode == ADAM) {
      h->m1.alloc((size_t)n_items); h->m2.alloc((size_t)n_items);
      B200_CUDA(cudaMemset(h->m1.get(), 0, sizeof(float) * (size_t)n_items));
      B200_CUDA(cudaMemset(h->m2.get(), 0, sizeof(float) * (size_t)n_items));
      p.m1 = h->m1.get(); p.m2 = h->m2.get();
    }
    h->su.alloc((size_t)n_users); h->si.alloc((size_t)n_users); h->sj.alloc((size_t)n_users);
    p.su = h->su.get(); p.si = h->si.get(); p.sj = h->sj.get();
    h->pow_out.alloc(2);
    p.pow_out = h->pow_out.get();
    B200_CUDA(cudaEventCreate(&h->ev0));
    B200_CUDA(cudaEventCreate(&h->ev1));
    *out = h;
  });
  if (rc != B200_OK && h) delete h;
  return rc;
}

int b200_slim_shard_partial_device(b200_slim_t h, int64_t first, int n_batch, float* d_x, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h && d_x && h->shard_hi > h->shard_lo, "b200_slim_shard_partial: not a sharded handle");
    B200_REQUIRE(first >= 0 && n_batch > 0 && first + n_batch <= h->p.n_users, "b200_slim_shard_partial: batch [%lld, +%d) outside the epoch",
                 (long long)first, n_batch);
    cudaStream_t st = (cudaStream_t)stream;
    if (h->drawn_epoch != (long long)h->epoch) {  // the epoch's whole stream, identical on every rank
      slim_sample_kernel<<<div_up(h->p.n_users, 256), 256, 0, st>>>(h->p.indptr, h->p.indices, h->p.n_users, h->p.n_items, h->p.n_users,
                                                                  h->seed, h->epoch, h->su.get(), h->si.get(), h->sj.get());
      count_launch();
      h->drawn_epoch = (long long)h->epoch;
    }
    ShardParams sp{h->p, h->shard_lo, h->shard_hi, h->shard_hi - h->shard_lo, (long long)first, n_batch};
    slim_shard_partial_kernel<<<std::min<int>(div_up(n_batch, 8), sm_count() * 8), 256, 0, st>>>(sp, d_x);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_slim_shard_apply_device(b200_slim_t h, int64_t first, int n_batch, const float* d_x_sum, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h && d_x_sum && h->shard_hi > h->shard_lo, "b200_slim_shard_apply: not a sharded handle");
    B200_REQUIRE(first >= 0 && n_batch > 0 && first + n_batch <= h->p.n_users && h->drawn_epoch == (long long)h->epoch,
                 "b200_slim_shard_apply: no partial step for this batch");
    ShardParams sp{h->p, h->shard_lo, h->shard_hi, h->shard_hi - h->shard_lo, (long long)first, n_batch};
    slim_shard_apply_kernel<<<std::min<int>(div_up(n_batch, 8), sm_count() * 8), 256, 0, (cudaStream_t)stream>>>(sp, d_x_sum);
    B200_CUDA(cudaGetLastError());
    count_launch();
    if (h->p.sgd_mode != SGD) {
      slim_shard_state_kernel<<<div_up(n_batch, 256), 256, 0, (cudaStream_t)stream>>>(sp, d_x_sum);
      B200_CUDA(cudaGetLastError());
      count_launch();
    }
    if (first + n_batch == h->p.n_users) {  // the epoch is complete
      if (h->p.sgd_mode == ADAM) {
        h->p.b1_pow *= pow((double)h->p.beta1, (double)h->p.n_users);
        h->p.b2_pow *= pow((double)h->p.beta2, (double)h->p.n_users);
      }
      h->epoch += 1;
    }
  });
}

int b200_slim_shard_device(b200_slim_t h, float** d_S, int* col_lo, int* col_hi) {
  return guarded([&] {
    B200_REQUIRE(h && h->shard_hi > h->shard_lo, "b200_slim_shard_device: not a sharded handle");
    if (d_S) *d_S = h->p.S;
    if (col_lo) *col_lo = h->shard_lo;
    if (col_hi) *col_hi = h->shard_hi;
  });
}

int b200_slim_destroy(b200_slim_t h) {
  if (!h) return B200_OK;
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
  return B200_OK;
}

int b200_slim_epoch(b200_slim_t h, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_slim_epoch: NULL handle");
    B200_REQUIRE(h->shard_hi == 0, "b200_slim_epoch: a column-sharded handle steps through b200_slim_shard_partial / _apply");
    cudaStream_t st = (cudaStream_t)stream;
    Params& p = h->p;
    const long long n = p.n_users;  // pyx:231: n_users samples per epoch
    p.n_samples = n;
    p.prof = getenv("B200REC_SLIM_PROF") != nullptr;
    if (h->sampler == 0) {
      h->hs_u.resize((size_t)n); h->hs_i.resize((size_t)n); h->hs_j.resize((size_t)n);
      const int* indptr = h->h_indptr.data();
      const int* indices = h->h_indices.data();
      for (long long g = 0; g < n; ++g) {  // sampleBPR_Cython pyx:436-480, draw for draw
        long u = 0, start = 0, len = 0;
        while (len == 0 || len == p.n_items) {
          u = h->rng.next() % p.n_users;
          start = indptr[u];
          len = indptr[u + 1] - start;
        }
        const long item = indices[start + h->rng.next() % len];
        long neg;
        for (;;) {
          neg = h->rng.next() % p.n_items;
          const int* lo = std::lower_bound(indices + start, indices + start + len, (int)neg);
          if (lo == indices + start + len || *lo != neg) break;
        }
        h->hs_u[(size_t)g] = (int)u; h->hs_i[(size_t)g] = (int)item; h->hs_j[(size_t)g] = (int)neg;
      }
      B200_CUDA(cudaMemcpyAsync(h->su.get(), h->hs_u.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
      B200_CUDA(cudaMemcpyAsync(h->si.get(), h->hs_i.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
      B200_CUDA(cudaMemcpyAsync(h->sj.get(), h->hs_j.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    }
    B200_CUDA(cudaEventRecord(h->ev0, st));
    if (h->sampler != 0) {
      slim_sample_kernel<<<div_up(n, 256), 256, 0, st>>>(p.indptr, p.indices, p.n_users, p.n_items, n, h->seed, h->epoch,
                                                        h->su.get(), h->si.get(), h->sj.get());
      count_launch();
    }
    if (h->hogwild) {
      slim_hogwild_kernel<<<sm_count() * 8, 256, 0, st>>>(p);
      if (p.sgd_mode == ADAM) { p.b1_pow *= pow((double)p.beta1, (double)n); p.b2_pow *= pow((double)p.beta2, (double)n); }
    } else if (h->tree) {
      // pyx:318-319: after sample n (n != 0) with `n % (n_users / 5) == 0` -- a float modulo under language_level=3 -- the rows
      // are cut back to their TopK; the epoch runs as the segments between those points
      long long first = 0;
      int launches = 0;
      const double period = (double)p.n_users / 5.0;
      for (long long g = 1; g <= n; ++g) {
        const bool prune_here = g < n && fmod((double)g, period) == 0.0;
        if (!prune_here && g != n) continue;
        const long long last = g < n ? g : n - 1;  // the segment ends with sample `last`
        Params q = p;
        q.first = first; q.n_samples = last - first + 1; q.chain_pow = first > 0;
        if (q.n_samples > 0) { slim_sequential_kernel<<<1, SEQ_THREADS, 0, st>>>(q); ++launches; }
        if (prune_here && h->tree_topk > 0) {
          slim_tree_prune_kernel<<<std::min(p.n_items, sm_count() * 8), 256, 0, st>>>(p.S, p.exists, p.n_items, h->tree_topk, 0);
          ++launches;
        }
        first = last + 1;
        if (g == n) break;
      }
      if (launches > 1) count_launch(launches - 1);  // the last one is counted below
    } else {
      slim_sequential_kernel<<<1, SEQ_THREADS, 0, st>>>(p);
    }
    B200_CUDA(cudaGetLastError());
    count_launch();
    B200_CUDA(cudaEventRecord(h->ev1, st));
    h->timed = true;
    if (!h->hogwild && p.sgd_mode == ADAM) {
      double pw[2];
      B200_CUDA(cudaMemcpyAsync(pw, h->pow_out.get(), sizeof(pw), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      p.b1_pow = pw[0]; p.b2_pow = pw[1];
    } else if (h->sampler == 0) {
      B200_CUDA(cudaStreamSynchronize(st));
    }
    h->epoch += 1;
  });
}

int b200_slim_enable_tree(b200_slim_t h, int topK) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_slim_enable_tree: NULL handle");
    B200_REQUIRE(h->shard_hi == 0 && !h->hogwild && !h->p.symmetric,
                 "b200_slim_enable_tree: the tree mode is sequential, non-symmetric (pyx:111-112) and single-GPU");
    B200_REQUIRE(h->epoch == 0 && !h->tree, "b200_slim_enable_tree: call once, before the first epoch");
    B200_REQUIRE(topK >= 0, "b200_slim_enable_tree: topK must be >= 0 (0 = False: rows are never cut)");
    const size_t cells = (size_t)h->p.n_items * (size_t)h->p.n_items;
    h->exists.alloc(cells);
    B200_CUDA(cudaMemset(h->exists.get(), 0, cells));
    h->p.exists = h->exists.get();
    h->tree = true;
    h->tree_topk = std::min(topK, h->p.n_items);
  });
}

int b200_slim_tree_prune(b200_slim_t h, int touch_diagonal, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr && h->tree, "b200_slim_tree_prune: not a tree-mode handle");
    const int n = h->p.n_items;
    slim_tree_prune_kernel<<<std::min(n, sm_count() * 8), 256, 0, (cudaStream_t)stream>>>(h->p.S, h->p.exists, n, h->tree_topk,
                                                                                           touch_diagonal != 0);
    B200_CUDA(cudaGetLastError());
    count_launch();
  });
}

int b200_slim_get_samples(b200_slim_t h, int32_t* u, int32_t* i, int32_t* j) {
  return guarded([&] {
    B200_REQUIRE(h && u && i && j, "b200_slim_get_samples: NULL argument");
    B200_CUDA(cudaDeviceSynchronize());
    const size_t n = (size_t)h->p.n_users;
    B200_CUDA(cudaMemcpy(u, h->su.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
    B200_CUDA(cudaMemcpy(i, h->si.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
    B200_CUDA(cudaMemcpy(j, h->sj.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
  });
}

int b200_slim_get_S_dense(b200_slim_t h, float* h_out, float* d_out) {
  return guarded([&] {
    B200_REQUIRE(h && (h_out || d_out), "b200_slim_get_S_dense: NULL argument");
    B200_REQUIRE(h->shard_hi == 0, "b200_slim_get_S_dense: a column-sharded handle exposes its slab through b200_slim_shard_device");
    const int n = h->p.n_items;
    const size_t cells = (size_t)n * n;
    DevBuf<float> tmp;
    float* dst = d_out;
    if (!dst) { tmp.alloc(cells); dst = tmp.get(); }
    // the epoch kernels run on the caller's stream (possibly a non-blocking one) and need not have finished: this entry
    // point has no stream argument, so it waits for the whole device before it reads S on the default stream
    B200_CUDA(cudaDeviceSynchronize());
    slim_full_kernel<<<div_up((long long)cells, 256), 256>>>(h->p.S, n, h->p.symmetric, dst);
    B200_CUDA(cudaGetLastError());
    count_launch();
    if (h_out) B200_CUDA(cudaMemcpy(h_out, dst, cells * sizeof(float), cudaMemcpyDeviceToHost));
    else B200_CUDA(cudaDeviceSynchronize());
  });
}

int b200_slim_last_epoch_ms(b200_slim_t h, float* ms) {
  return guarded([&] {
    B200_REQUIRE(h && ms && h->timed, "b200_slim_last_epoch_ms: no epoch run yet");
    B200_CUDA(cudaEventSynchronize(h->ev1));
    B200_CUDA(cudaEventElapsedTime(ms, h->ev0, h->ev1));
  });
}

}  // extern "C"
