// K3: SLIM-BPR epochs on a dense (optionally symmetric) item-item matrix S, sm_90a.
//
// Replaces SLIM_BPR/Cython/SLIM_BPR_Cython_Epoch.pyx: epochIteration_Cython :211-335, sampleBPR_Cython :436-480,
// adaptive_gradient :395-433 (per-ITEM scalar state shared by the positive and negative roles), symmetric storage
// Triangular_Matrix :1272-1330, get_S :340-388 (diagonal zeroed).  S is dense fp32 in HBM (C2: 55 MB, L2-resident).
// The tree-sparse training mode (train_with_sparse_weights, Sparse_Matrix_Tree_CSR :579-1031) keeps S ROW-SPARSE: a
// row-sorted CSR of the cells the reference's row trees hold.  The sample stream of an epoch does not depend on S, so
// before a segment (the samples between two rebalance_tree(TopK) cuts, :318-319, :782-802) runs, the cells it will create
// are known: the structure is rebuilt with them (value 0, which is what a cell that does not exist yet reads), a slot map
// gives every update of the segment the index of its cell, and the sequential kernel runs on `val[slot]`.  The cut and the
// in-place selection of get_scipy_csr(TopK) :762-763 keep the K largest cells of each longer row.
//
// Two execution modes (DESIGN.md "K3"):
//   * sequential (the reference's semantics exactly): the recursion is batch-1 and every sample reads cells the
//     previous one may have written, so ONE CTA walks the replayed sample stream in order; the 2*len_u cell reads,
//     the x_uij reduction and the 2*len_u updates of a sample are spread over the CTA's threads.
//   * hogwild: all SMs, one warp per sample, float atomics on S (Hogwild races), Philox or replayed stream.
// Roofline: HBM/L2, 4*len_u*4 bytes per sample for S (two row gathers read + written) + 4*len_u for the profile.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "adaptive.cuh"
#include "common.cuh"
#include "sampler.cuh"
#include "select.cuh"

namespace b200 {
namespace slim {

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
  float* val;              // tree mode: the values of the row-sparse cells (TreeStore)
  const long long* slot_i; // tree mode: per update of the segment, in sample order, the cell of (i, s) (-1: s == i, never
  const long long* slot_j; //   written, reads 0) and of (j, s) in val
  long long first;         // first sample of this launch (tree mode runs an epoch as segments between two prunings)
  int chain_pow;           // continue the Adam powers from pow_out (segment > 0) instead of b1_pow / b2_pow
  int prof;                // B200REC_SLIM_PROF=1: thread 0 times the phases of the sequential kernel (development hook)
};

__device__ __forceinline__ size_t cell(const Params& p, int a, int b) {
  if (p.symmetric && b > a) { const int t = a; a = b; b = t; }  // pyx:1287-1302, 1309-1330
  return (size_t)a * p.n_items + b;
}

__device__ __forceinline__ float adapt_item(const Params& p, float g, int item, float inv1, float inv2) {  // pyx:395-433
  if (p.sgd_mode == B200_ADAGRAD) {
    const float cc = p.c[item] + g * g;
    p.c[item] = cc;
    return g / (sqrtf(cc) + 1e-8f);
  } else if (p.sgd_mode == B200_RMSPROP) {
    const float cc = p.c[item] * p.gamma + (1.f - p.gamma) * g * g;
    p.c[item] = cc;
    return g / (sqrtf(cc) + 1e-8f);
  } else if (p.sgd_mode == B200_ADAM) {
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
// CELLS is how a cell is addressed: DENSE_CELLS through cell(p, a, b) in S; SLOT_CELLS (tree mode) through the segment's
// slot map into val, with the same thread <-> profile-entry mapping and reduction order, so the fp32 arithmetic is the same.
enum CellAddr { DENSE_CELLS = 0, SLOT_CELLS = 1 };
template <int CELLS>
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
  // sample n in (u, i, j, s, e, sn0); sample n + 1 in (nu, ni, nj).  SLOT_CELLS: the slots of this thread's entry of
  // sample n in (ci0, cj0) (cj0 = -1: no entry), the sample's first update at `base` of the slot map
  int u = 0, i = 0, j = 0, s = 0, e = 0, sn0 = -1, nu = 0, ni = 0, nj = 0;
  long long base = 0, ci0 = -1, cj0 = -1;
  if (p.n_samples > 0) {
    u = p.su[p.first]; i = p.si[p.first]; j = p.sj[p.first];
    s = p.indptr[u]; e = p.indptr[u + 1];
    if constexpr (CELLS == DENSE_CELLS) {
      if (s + tid < e) sn0 = p.indices[s + tid];
    } else {
      if (s + tid < e) { ci0 = p.slot_i[tid]; cj0 = p.slot_j[tid]; }
    }
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
      if (p.sgd_mode == B200_ADAGRAD || p.sgd_mode == B200_RMSPROP) { st_i0 = p.c[i]; st_j0 = p.c[j]; }
      else if (p.sgd_mode == B200_ADAM) { st_i0 = p.m1[i]; st_i1 = p.m2[i]; st_j0 = p.m1[j]; st_j1 = p.m2[j]; }
    }
    float x = 0.f;
    int nsn0 = -1;
    long long nci0 = -1, ncj0 = -1;
    const long long nbase = base + (e - s);
    if constexpr (CELLS == DENSE_CELLS) {
      if (sn0 >= 0) x = p.S[cell(p, i, sn0)] - p.S[cell(p, j, sn0)];  // pyx:242-255
      for (int k = s + tid + SEQ_THREADS; k < e; k += SEQ_THREADS) {
        const int sn = p.indices[k];
        x += p.S[cell(p, i, sn)] - p.S[cell(p, j, sn)];
      }
      if (ns + tid < ne) nsn0 = p.indices[ns + tid];  // the next sample's profile entry of this thread
    } else {
      if (cj0 >= 0) x = (ci0 >= 0 ? p.val[ci0] : 0.f) - p.val[cj0];
      for (long long q = base + tid + SEQ_THREADS; q < nbase; q += SEQ_THREADS) {
        const long long a = p.slot_i[q];
        x += (a >= 0 ? p.val[a] : 0.f) - p.val[p.slot_j[q]];
      }
      if (n + 1 < last && ns + tid < ne) { nci0 = p.slot_i[nbase + tid]; ncj0 = p.slot_j[nbase + tid]; }  // the next sample's slots
    }
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
        const float inv1 = adam_correction(b1p), inv2 = adam_correction(b2p);
        float gi = g, gj = g;  // i first, then j (pyx:262-263); i != j always (j is not in the profile, i is)
        if (p.sgd_mode == B200_ADAGRAD) {
          st_i0 += g * g; gi = g / (sqrtf(st_i0) + 1e-8f); p.c[i] = st_i0;
          st_j0 += g * g; gj = g / (sqrtf(st_j0) + 1e-8f); p.c[j] = st_j0;
        } else if (p.sgd_mode == B200_RMSPROP) {
          st_i0 = st_i0 * p.gamma + (1.f - p.gamma) * g * g; gi = g / (sqrtf(st_i0) + 1e-8f); p.c[i] = st_i0;
          st_j0 = st_j0 * p.gamma + (1.f - p.gamma) * g * g; gj = g / (sqrtf(st_j0) + 1e-8f); p.c[j] = st_j0;
        } else if (p.sgd_mode == B200_ADAM) {
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
    if constexpr (CELLS == DENSE_CELLS) {
      for (int k = s + tid; k < e; k += SEQ_THREADS) {
        const int sn = k == s + tid ? sn0 : p.indices[k];
        if (sn != i) { const size_t c = cell(p, i, sn); const float v = p.S[c]; p.S[c] = v + p.lr * (gi - p.li_reg * v); }
        if (sn != j) { const size_t c = cell(p, j, sn); const float v = p.S[c]; p.S[c] = v - p.lr * (gj - p.lj_reg * v); }
      }
    } else {
      for (long long q = base + tid; q < nbase; q += SEQ_THREADS) {
        const long long a = q == base + tid ? ci0 : p.slot_i[q];
        const long long b = q == base + tid ? cj0 : p.slot_j[q];
        if (a >= 0) { const float v = p.val[a]; p.val[a] = v + p.lr * (gi - p.li_reg * v); }
        { const float v = p.val[b]; p.val[b] = v - p.lr * (gj - p.lj_reg * v); }  // s != j: j is not in the profile
      }
    }
    if (p.sgd_mode == B200_ADAM) { b1p *= (double)p.beta1; b2p *= (double)p.beta2; }  // per sample, pyx:309-312
    u = nu; i = ni; j = nj; s = ns; e = ne; sn0 = nsn0;
    base = nbase; ci0 = nci0; cj0 = ncj0;
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
    if (p.sgd_mode != B200_SGD) {
      float inv1 = 1.f, inv2 = 1.f;
      if (p.sgd_mode == B200_ADAM) {
        inv1 = adam_correction(p.b1_pow * pow((double)p.beta1, (double)n));
        inv2 = adam_correction(p.b2_pow * pow((double)p.beta2, (double)n));
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
  if (p.sgd_mode == B200_ADAGRAD) return g / (sqrtf(p.c[item] + g * g) + 1e-8f);
  if (p.sgd_mode == B200_RMSPROP) return g / (sqrtf(p.c[item] * p.gamma + (1.f - p.gamma) * g * g) + 1e-8f);
  if (p.sgd_mode == B200_ADAM) {
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
    if (p.sgd_mode != B200_SGD) {
      float inv1 = 1.f, inv2 = 1.f;
      if (p.sgd_mode == B200_ADAM) {  // the powers advance once per sample (pyx:309-312)
        inv1 = adam_correction(p.b1_pow * pow((double)p.beta1, (double)g));
        inv2 = adam_correction(p.b2_pow * pow((double)p.beta2, (double)g));
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
    if (p.sgd_mode == B200_ADAGRAD) atomicAdd(p.c + it, gr * gr);
    else if (p.sgd_mode == B200_RMSPROP) ema_atomic(p.c + it, p.gamma, (1.f - p.gamma) * gr * gr);
    else if (p.sgd_mode == B200_ADAM) { ema_atomic(p.m1 + it, p.beta1, (1.f - p.beta1) * gr); ema_atomic(p.m2 + it, p.beta2, (1.f - p.beta2) * gr * gr); }
  }
}

// ---- tree mode (row-sparse).  The cells live in a row-sorted CSR: key[t] = (row << 32) | col, val[t], rowptr[n + 1].
// Per segment: (1) structure: the cells kept so far plus every cell the segment touches (row i gains profile(u) \ {i}, row j
// gains profile(u)) are radix-sorted and de-duplicated; kept cells keep their value, new ones start at 0 -- what a cell that
// does not exist yet reads in the reference; (2) slot map: per update, in sample order, the index of its cell; (3) values:
// slim_sequential_kernel<SLOT_CELLS>; (4) cut: rows holding more than K cells keep their K largest.
typedef unsigned long long u64;
__device__ __forceinline__ u64 tree_cell_key(int r, int c) { return ((u64)(unsigned)r << 32) | (u64)(unsigned)c; }

// one warp per sample of the segment: 2 * len_u keys at 2 * (off[n] - off[first]).  The (i, i) update is never made (s == i),
// so its place holds a second copy of (j, i), which the de-duplication removes.
__global__ void __launch_bounds__(256) slim_tree_touch_kernel(const Params p, const long long* __restrict__ off, u64* out) {
  const int lane = threadIdx.x & 31;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long off0 = off[p.first];
  for (long long g = w; g < p.n_samples; g += n_warps) {
    const long long n = p.first + g;
    const int u = p.su[n], i = p.si[n], j = p.sj[n];
    const int s = p.indptr[u], len = p.indptr[u + 1] - s;
    u64* o = out + 2 * (off[n] - off0);
    for (int k = lane; k < len; k += 32) {
      const int sn = p.indices[s + k];
      o[k] = sn == i ? tree_cell_key(j, sn) : tree_cell_key(i, sn);
      o[len + k] = tree_cell_key(j, sn);
    }
  }
}

__global__ void slim_tree_diag_kernel(int n, u64* out) {  // get_S touches (r, r), pyx:349-350
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = tree_cell_key(r, r);
}

// rowptr of m sorted unique keys: the first cell of row r is the first key whose row is >= r
__global__ void slim_tree_rowptr_kernel(const u64* __restrict__ key, long long m, int n, long long* rowptr) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > m) return;
  const int r = t < m ? (int)(key[t] >> 32) : n;
  const int rp = t > 0 ? (int)(key[t - 1] >> 32) : -1;
  for (int q = rp + 1; q <= r; ++q) rowptr[q] = t;
}

__device__ __forceinline__ long long tree_find(const u64* __restrict__ key, long long lo, long long hi, u64 k) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (key[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the new structure's values: the old value of a cell that existed before, 0 for a new one
__global__ void slim_tree_carry_kernel(const u64* __restrict__ key, long long m, const u64* __restrict__ old_key,
                                       const float* __restrict__ old_val, const long long* __restrict__ old_rowptr, float* val) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const u64 k = key[t];
  const int r = (int)(k >> 32);
  const long long lo = old_rowptr[r], hi = old_rowptr[r + 1];
  const long long q = tree_find(old_key, lo, hi, k);
  val[t] = q < hi && old_key[q] == k ? old_val[q] : 0.f;
}

// one warp per sample: the cells of its 2 * len_u updates in the new structure
__global__ void __launch_bounds__(256) slim_tree_slot_kernel(const Params p, const long long* __restrict__ off, const u64* __restrict__ key,
                                                             const long long* __restrict__ rowptr, long long* slot_i, long long* slot_j) {
  const int lane = threadIdx.x & 31;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long off0 = off[p.first];
  for (long long g = w; g < p.n_samples; g += n_warps) {
    const long long n = p.first + g;
    const int u = p.su[n], i = p.si[n], j = p.sj[n];
    const int s = p.indptr[u], len = p.indptr[u + 1] - s;
    const long long q0 = off[n] - off0;
    const long long ilo = rowptr[i], ihi = rowptr[i + 1], jlo = rowptr[j], jhi = rowptr[j + 1];
    for (int k = lane; k < len; k += 32) {
      const int sn = p.indices[s + k];
      slot_i[q0 + k] = sn == i ? -1 : tree_find(key, ilo, ihi, tree_cell_key(i, sn));
      slot_j[q0 + k] = tree_find(key, jlo, jhi, tree_cell_key(j, sn));
    }
  }
}

// ---- the cut: rebalance_tree(TopK) pyx:782-802 and the in-place selection inside get_scipy_csr(TopK) pyx:762-763, both
// through topK_selection_from_list pyx:954-1031.  A row holding more than K cells keeps the K largest by value; the reference
// sorts the column-ordered list with a stable qsort on the value, so among equal values the HIGHER columns survive:
// key = (orderable value << 32) | column, keep the K largest keys.  Dropped cells vanish from the structure (a later touch
// creates them again with value 0).  One warp per row: radix select (select.cuh, 8-bit digits) over the 64-bit keys, read
// from the row in global memory (L1/L2-resident across the passes).
__device__ __forceinline__ u64 tree_cut_key(u64 cell, float v) { return ((u64)orderable(v) << 32) | (cell & 0xFFFFFFFFull); }

constexpr int CUT_THREADS = 256;
// thr[r]: the row keeps the cells whose cut key is >= thr[r]; cnt[r]: how many
__global__ void __launch_bounds__(CUT_THREADS) slim_tree_cut_select_kernel(const u64* __restrict__ key, const float* __restrict__ val,
                                                                           const long long* __restrict__ rowptr, int n, int K, u64* thr,
                                                                           long long* cnt) {
  __shared__ __align__(16) int hist[CUT_THREADS / 32][256];
  const int lane = threadIdx.x & 31;
  const WarpSelect g{hist[threadIdx.x >> 5]};
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int n_warps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int row = w; row < n; row += n_warps) {
    const long long lo = rowptr[row], hi = rowptr[row + 1];
    if (hi - lo <= K) {  // fewer than K cells: the list is returned as it is (pyx:977-978); exactly K: all stay
      if (lane == 0) { thr[row] = 0ull; cnt[row] = hi - lo; }
      continue;
    }
    const auto sel_key = [&](int q, u64& k) {
      k = tree_cut_key(key[lo + q], val[lo + q]);
      return true;
    };
    const u64 t = radix_select<u64, 8, false>(g, (int)(hi - lo), K, sel_key).thr;
    if (lane == 0) { thr[row] = t; cnt[row] = K; }
  }
}

// the kept cells, in column order, into the new structure at rowptr_new
__global__ void __launch_bounds__(CUT_THREADS) slim_tree_cut_compact_kernel(const u64* __restrict__ key, const float* __restrict__ val,
                                                                            const long long* __restrict__ rowptr, int n,
                                                                            const u64* __restrict__ thr, const long long* __restrict__ rowptr_new,
                                                                            u64* key_new, float* val_new) {
  const int lane = threadIdx.x & 31;
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int n_warps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int row = w; row < n; row += n_warps) {
    const long long lo = rowptr[row], hi = rowptr[row + 1];
    const u64 T = thr[row];
    long long dst = rowptr_new[row];
    for (long long b = lo; b < hi; b += 32) {
      const long long t = b + lane;
      u64 k = 0; float v = 0.f;
      bool keep = false;
      if (t < hi) { k = key[t]; v = val[t]; keep = tree_cut_key(k, v) >= T; }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const long long d = dst + __popc(bal & ((1u << lane) - 1u));
        key_new[d] = k; val_new[d] = v;
      }
      dst += __popc(bal);
    }
  }
}

// CSR export of the non-zero off-diagonal cells: per-row counts, then (after a scan) the fill
__global__ void __launch_bounds__(256) slim_tree_export_kernel(const u64* __restrict__ key, const float* __restrict__ val,
                                                               const long long* __restrict__ rowptr, int n, long long* cnt,
                                                               const long long* __restrict__ out_ptr, int* out_idx, float* out_val) {
  const int lane = threadIdx.x & 31;
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int n_warps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int row = w; row < n; row += n_warps) {
    const long long lo = rowptr[row], hi = rowptr[row + 1];
    long long dst = out_ptr ? out_ptr[row] : 0;
    for (long long b = lo; b < hi; b += 32) {
      const long long t = b + lane;
      int c = 0; float v = 0.f;
      bool keep = false;
      if (t < hi) { c = (int)(unsigned)key[t]; v = val[t]; keep = v != 0.f && c != row; }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (out_ptr && keep) {
        const long long d = dst + __popc(bal & ((1u << lane) - 1u));
        out_idx[d] = c; out_val[d] = v;
      }
      dst += __popc(bal);
    }
    if (!out_ptr && lane == 0) cnt[row] = dst;
  }
}

// the raw tree state as the dense view get_S starts from (diagonal 0) into a zeroed n x n buffer
__global__ void tree_len_kernel(const int* __restrict__ su, const int* __restrict__ indptr, long long n, long long* len) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) { const int u = su[g]; len[g] = indptr[u + 1] - indptr[u]; }
  else if (g == n) len[g] = 0;
}

__global__ void slim_tree_scatter_kernel(const u64* __restrict__ key, const float* __restrict__ val, long long m, int n, float* out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const u64 k = key[t];
  const int r = (int)(k >> 32), c = (int)(unsigned)k;
  if (r != c) out[(size_t)r * n + c] = val[t];
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

// grows a scratch buffer to at least `count` elements (contents are not kept)
template <typename T>
void reserve(DevBuf<T>& b, size_t count) {
  if (b.n < count) b.alloc(count + count / 4);
}

// the row-sparse tree state and the per-segment scratch
struct TreeStore {
  DevBuf<u64> key, key_new;            // row-sorted cells
  DevBuf<float> val, val_new;
  DevBuf<long long> rowptr, rowptr_new;  // n_items + 1
  long long m = 0;                       // cells in the structure
  DevBuf<u64> kin, kalt;                 // structure build: cells in, sorted
  DevBuf<long long> slot_i, slot_j;      // slot map of the running segment
  DevBuf<long long> len, off;            // per sample of the epoch: profile length and its exclusive prefix sum (n_users + 1)
  DevBuf<u64> thr;                       // cut: per row, the smallest kept key
  DevBuf<long long> cnt, count;          // cut / export: per-row counts (n_items + 1); de-duplicated key count
  DevBuf<unsigned char> tmp;             // CUB scratch

  void* scratch(size_t bytes) { reserve(tmp, std::max<size_t>(bytes, 1)); return tmp.get(); }

  // rowptr_new from cnt[0, n) (cnt[n] = 0)
  void scan_counts(int n, cudaStream_t st) {
    size_t tb = 0;
    B200_CUDA(cudaMemsetAsync(cnt.get() + n, 0, sizeof(long long), st));
    B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.get(), rowptr_new.get(), n + 1, st));
    B200_CUDA(cub::DeviceScan::ExclusiveSum(scratch(tb), tb, cnt.get(), rowptr_new.get(), n + 1, st));
    count_launch();
  }

  // (1) the structure: the current cells merged with `extra` new keys that `emit` writes after them.  One host read.
  template <typename Emit>
  void build(int n, long long extra, cudaStream_t st, Emit emit) {
    const long long total = m + extra;
    reserve(kin, (size_t)total); reserve(kalt, (size_t)total); reserve(key_new, (size_t)total); reserve(val_new, (size_t)total);
    if (m) B200_CUDA(cudaMemcpyAsync(kin.get(), key.get(), sizeof(u64) * (size_t)m, cudaMemcpyDeviceToDevice, st));
    emit(kin.get() + m);
    int bits = 1;
    while ((1ll << bits) <= (long long)n) ++bits;
    cub::DoubleBuffer<u64> db(kin.get(), kalt.get());
    size_t tb = 0, tb2 = 0;
    B200_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, total, 0, 32 + bits, st));
    B200_CUDA(cub::DeviceSelect::Unique(nullptr, tb2, db.Current(), key_new.get(), count.get(), total, st));
    void* t = scratch(std::max(tb, tb2));
    B200_CUDA(cub::DeviceRadixSort::SortKeys(t, tb, db, total, 0, 32 + bits, st));
    B200_CUDA(cub::DeviceSelect::Unique(t, tb2, db.Current(), key_new.get(), count.get(), total, st));
    long long m_new = 0;
    B200_CUDA(cudaMemcpyAsync(&m_new, count.get(), sizeof(long long), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    slim_tree_rowptr_kernel<<<div_up(m_new + 1, 256), 256, 0, st>>>(key_new.get(), m_new, n, rowptr_new.get());
    if (m_new) slim_tree_carry_kernel<<<div_up(m_new, 256), 256, 0, st>>>(key_new.get(), m_new, key.get(), val.get(), rowptr.get(), val_new.get());
    B200_CUDA(cudaGetLastError());
    count_launch(4);
    std::swap(key, key_new); std::swap(val, val_new); std::swap(rowptr, rowptr_new);
    m = m_new;
  }

  // (4) rows holding more than K cells keep their K largest.  One host read.
  void cut(int n, int K, cudaStream_t st) {
    const int grid = std::min<int>(div_up(n, CUT_THREADS / 32), sm_count() * 16);
    slim_tree_cut_select_kernel<<<grid, CUT_THREADS, 0, st>>>(key.get(), val.get(), rowptr.get(), n, K, thr.get(), cnt.get());
    B200_CUDA(cudaGetLastError());
    scan_counts(n, st);
    long long m_new = 0;
    B200_CUDA(cudaMemcpyAsync(&m_new, rowptr_new.get() + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    reserve(key_new, (size_t)std::max(m_new, 1ll)); reserve(val_new, (size_t)std::max(m_new, 1ll));
    slim_tree_cut_compact_kernel<<<grid, CUT_THREADS, 0, st>>>(key.get(), val.get(), rowptr.get(), n, thr.get(), rowptr_new.get(),
                                                                key_new.get(), val_new.get());
    B200_CUDA(cudaGetLastError());
    count_launch(2);
    std::swap(key, key_new); std::swap(val, val_new); std::swap(rowptr, rowptr_new);
    m = m_new;
  }
};

}  // namespace slim
}  // namespace b200

using namespace b200;
using namespace b200::slim;

struct b200_slim_s {
  Params p{};
  SampleStream ss;
  int hogwild = 0;
  unsigned seed = 1, epoch = 0;
  DevBuf<float> S;
  AdaptBuffers state;  // per item
  DevBuf<double> pow_out;
  EpochTimer timer;
  int shard_lo = 0, shard_hi = 0;  // column-sharded handle (b200_slim_create_sharded): S is [n_items, shard_hi - shard_lo]
  long long drawn_epoch = -1;      // the epoch whose sample stream is in su / si / sj
  TreeStore ts;                    // tree mode (b200_slim_enable_tree)
  bool tree = false;
  int tree_topk = 0;
};

// the dense S of a non-tree handle, allocated (zeroed: pyx:122-125) by the first call that needs it
static void ensure_dense_S(b200_slim_s* h, cudaStream_t st) {
  if (h->S.get()) return;
  const int n = h->p.n_items;
  B200_REQUIRE((double)n * (double)n * 4.0 < 1.6e11, "b200_slim_create: dense S does not fit one GPU");
  const size_t cells = (size_t)n * (size_t)n;
  h->S.alloc(cells);
  B200_CUDA(cudaMemsetAsync(h->S.get(), 0, cells * sizeof(float), st));
  h->p.S = h->S.get();
}

// pyx:318-319: after sample n (n != 0) with `n % (n_users / 5) == 0` -- a float modulo under language_level=3 -- the rows
// are cut back to their TopK; the epoch runs as the segments between those points, each on the structure built for it
static void tree_epoch(b200_slim_s* h, cudaStream_t st) {
  Params& p = h->p;
  TreeStore& T = h->ts;
  const long long n = p.n_users;
  const int ni = p.n_items;
  // off[g] = sum of the profile lengths of samples < g
  tree_len_kernel<<<div_up(n + 1, 256), 256, 0, st>>>(p.su, p.indptr, n, T.len.get());
  size_t tb = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, T.len.get(), T.off.get(), n + 1, st));
  B200_CUDA(cub::DeviceScan::ExclusiveSum(T.scratch(tb), tb, T.len.get(), T.off.get(), n + 1, st));
  int launches = 2;
  struct Seg { long long first, last; bool cut; };
  std::vector<Seg> segs;
  long long first = 0;
  const double period = (double)p.n_users / 5.0;
  for (long long g = 1; g <= n; ++g) {
    const bool prune_here = g < n && fmod((double)g, period) == 0.0;
    if (!prune_here && g != n) continue;
    const long long last = g < n ? g : n - 1;  // the segment ends with sample `last`
    segs.push_back({first, last, prune_here});
    first = last + 1;
    if (g == n) break;
  }
  std::vector<long long> bounds(segs.size() + 1);
  for (size_t k = 0; k < segs.size(); ++k)
    B200_CUDA(cudaMemcpyAsync(&bounds[k], T.off.get() + segs[k].first, sizeof(long long), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(&bounds[segs.size()], T.off.get() + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  for (size_t k = 0; k < segs.size(); ++k) {
    Params q = p;
    q.first = segs[k].first; q.n_samples = segs[k].last - segs[k].first + 1; q.chain_pow = segs[k].first > 0;
    const long long updates = bounds[k + 1] - bounds[k];
    if (q.n_samples > 0) {  // every sampled profile is non-empty (pyx:443-447): updates > 0
      const unsigned grid = std::min<long long>(div_up(q.n_samples, 8), (long long)sm_count() * 16);
      T.build(ni, 2 * updates, st, [&](u64* out) {
        slim_tree_touch_kernel<<<grid, 256, 0, st>>>(q, T.off.get(), out);
      });
      reserve(T.slot_i, (size_t)updates); reserve(T.slot_j, (size_t)updates);
      slim_tree_slot_kernel<<<grid, 256, 0, st>>>(q, T.off.get(), T.key.get(), T.rowptr.get(), T.slot_i.get(), T.slot_j.get());
      q.val = T.val.get(); q.slot_i = T.slot_i.get(); q.slot_j = T.slot_j.get();
      slim_sequential_kernel<SLOT_CELLS><<<1, SEQ_THREADS, 0, st>>>(q);
      B200_CUDA(cudaGetLastError());
      launches += 3;
    }
    if (segs[k].cut && h->tree_topk > 0) T.cut(ni, h->tree_topk, st);
  }
  count_launch(launches - 1);  // the last one is counted by the caller
}

// The body of b200_slim_create and b200_slim_create_sharded: every check before any CUDA call, then the handle.  A sharded
// handle holds the columns [col_lo, col_hi) of S from the start; a single-GPU one allocates S when a call first needs it
// (ensure_dense_S), so a handle that becomes a tree handle (b200_slim_enable_tree) never holds one.
static int create(const char* fn, b200_slim_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                  const int32_t* h_indices, float learning_rate, float li_reg, float lj_reg, int symmetric, int sgd_mode, float gamma,
                  float beta_1, float beta_2, uint32_t seed, int sampler, int hogwild, bool sharded, int col_lo, int col_hi) {
  if (out) *out = nullptr;
  b200_slim_s* h = nullptr;
  int rc = guarded([&] {
    B200_REQUIRE(out && h_indptr && (nnz == 0 || h_indices), "%s: NULL argument", fn);
    B200_REQUIRE(n_users > 0 && n_items > 0 && nnz >= 0 && nnz < (1ll << 31) - 1, "%s: bad shape", fn);
    B200_REQUIRE(sgd_mode >= B200_SGD && sgd_mode <= B200_ADAM, "%s: unknown sgd_mode %d", fn, sgd_mode);
    B200_REQUIRE(!sharded || (0 <= col_lo && col_lo < col_hi && col_hi <= n_items), "%s: bad column range [%d,%d)", fn, col_lo, col_hi);
    B200_REQUIRE(sampler == 0 || has_sampleable_user(h_indptr, 0, n_users, n_items),
                 "%s: no user has 0 < profile length < n_items, the device sampler cannot draw a sample", fn);
    h = new b200_slim_s();
    Params& p = h->p;
    p.n_users = (int)n_users; p.n_items = (int)n_items; p.symmetric = symmetric != 0; p.sgd_mode = sgd_mode;
    p.lr = learning_rate; p.li_reg = li_reg; p.lj_reg = lj_reg; p.gamma = gamma; p.beta1 = beta_1; p.beta2 = beta_2;
    p.b1_pow = beta_1; p.b2_pow = beta_2;  // pyx:157-158
    h->hogwild = hogwild != 0;
    h->seed = seed;
    h->shard_lo = col_lo; h->shard_hi = col_hi;
    h->ss.init(n_users, n_items, nnz, h_indptr, h_indices, nullptr, true, 0.0, (size_t)n_users, sampler != 0, 0x243F6A88u, seed, false);
    p.indptr = h->ss.indptr.get(); p.indices = h->ss.indices.get();
    p.su = h->ss.su.get(); p.si = h->ss.si.get(); p.sj = h->ss.sj.get();
    const AdaptState a = h->state.alloc(sgd_mode, (size_t)n_items);
    if (sgd_mode == B200_ADAM) p.m1 = a.s1; else p.c = a.s1;
    p.m2 = a.s2;
    if (sharded) {
      h->S.alloc_zeroed((size_t)n_items * (size_t)(col_hi - col_lo));  // pyx:122-125
      p.S = h->S.get();
    }
    h->pow_out.alloc(2);
    p.pow_out = h->pow_out.get();
    *out = h;
  });
  if (rc != B200_OK && h) delete h;
  return rc;
}

extern "C" {

int b200_slim_create(b200_slim_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                     const int32_t* h_indices, float learning_rate, float li_reg, float lj_reg, int symmetric, int sgd_mode,
                     float gamma, float beta_1, float beta_2, int has_seed, uint32_t random_seed, int sampler, int hogwild) {
  return create("b200_slim_create", out, n_users, n_items, nnz, h_indptr, h_indices, learning_rate, li_reg, lj_reg, symmetric,
                sgd_mode, gamma, beta_1, beta_2, has_seed ? random_seed : 1u, sampler, hogwild, false, 0, 0);
}

int b200_slim_create_sharded(b200_slim_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                             const int32_t* h_indices, float learning_rate, float li_reg, float lj_reg, int sgd_mode, float gamma,
                             float beta_1, float beta_2, uint32_t random_seed, int col_lo, int col_hi) {
  return create("b200_slim_create_sharded", out, n_users, n_items, nnz, h_indptr, h_indices, learning_rate, li_reg, lj_reg, 0, sgd_mode,
                gamma, beta_1, beta_2, random_seed, 1, 1, true, col_lo, col_hi);
}

int b200_slim_shard_partial_device(b200_slim_t h, int64_t first, int n_batch, float* d_x, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h && d_x && h->shard_hi > h->shard_lo, "b200_slim_shard_partial: not a sharded handle");
    B200_REQUIRE(first >= 0 && n_batch > 0 && first + n_batch <= h->p.n_users, "b200_slim_shard_partial: batch [%lld, +%d) outside the epoch",
                 (long long)first, n_batch);
    cudaStream_t st = (cudaStream_t)stream;
    if (h->drawn_epoch != (long long)h->epoch) {  // the epoch's whole stream, identical on every rank
      h->ss.draw_philox(h->p.n_users, h->seed, h->epoch, 0, h->p.n_users, st);
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
    if (h->p.sgd_mode != B200_SGD) {
      slim_shard_state_kernel<<<div_up(n_batch, 256), 256, 0, (cudaStream_t)stream>>>(sp, d_x_sum);
      B200_CUDA(cudaGetLastError());
      count_launch();
    }
    if (first + n_batch == h->p.n_users) {  // the epoch is complete
      if (h->p.sgd_mode == B200_ADAM) advance_powers(h->p.beta1, h->p.beta2, h->p.b1_pow, h->p.b2_pow, (double)h->p.n_users);
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
    h->ss.draw_glibc(n, st);
    h->timer.begin(st);
    h->ss.draw_philox(n, h->seed, h->epoch, 0, p.n_users, st);
    if (!h->tree) ensure_dense_S(h, st);
    if (h->hogwild) {
      slim_hogwild_kernel<<<sm_count() * 8, 256, 0, st>>>(p);
      if (p.sgd_mode == B200_ADAM) advance_powers(p.beta1, p.beta2, p.b1_pow, p.b2_pow, (double)n);
    } else if (h->tree) {
      tree_epoch(h, st);
    } else {
      slim_sequential_kernel<DENSE_CELLS><<<1, SEQ_THREADS, 0, st>>>(p);
    }
    B200_CUDA(cudaGetLastError());
    count_launch();
    h->timer.end(st);
    if (!h->hogwild && p.sgd_mode == B200_ADAM) {
      read_powers(h->pow_out.get(), p.b1_pow, p.b2_pow, st);
    } else if (h->ss.host_vectors_in_flight()) {
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
    const int n = h->p.n_items;
    TreeStore& T = h->ts;
    T.rowptr.alloc((size_t)n + 1); T.rowptr_new.alloc((size_t)n + 1);
    B200_CUDA(cudaMemset(T.rowptr.get(), 0, sizeof(long long) * ((size_t)n + 1)));  // no cells yet
    T.cnt.alloc((size_t)n + 1); T.thr.alloc((size_t)n); T.count.alloc(1);
    T.len.alloc((size_t)h->p.n_users + 1); T.off.alloc((size_t)h->p.n_users + 1);
    h->tree = true;
    h->tree_topk = std::min(topK, n);
  });
}

int b200_slim_tree_prune(b200_slim_t h, int touch_diagonal, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr && h->tree, "b200_slim_tree_prune: not a tree-mode handle");
    cudaStream_t st = (cudaStream_t)stream;
    const int n = h->p.n_items;
    TreeStore& T = h->ts;
    if (touch_diagonal)  // get_S: add_value(index, index, -get_value(index, index)), pyx:349-350 (the diagonal is never written)
      T.build(n, n, st, [&](u64* out) { slim_tree_diag_kernel<<<div_up(n, 256), 256, 0, st>>>(n, out); });
    if (h->tree_topk > 0) T.cut(n, h->tree_topk, st);
    B200_CUDA(cudaGetLastError());
  });
}

int b200_slim_tree_csr_nnz(b200_slim_t h, int64_t* nnz) {
  return guarded([&] {
    B200_REQUIRE(h && nnz && h->tree, "b200_slim_tree_csr_nnz: not a tree-mode handle");
    const int n = h->p.n_items;
    TreeStore& T = h->ts;
    B200_CUDA(cudaDeviceSynchronize());  // no stream argument: the epoch may still run on the caller's stream
    slim_tree_export_kernel<<<std::min<int>(div_up(n, 8), sm_count() * 16), 256>>>(T.key.get(), T.val.get(), T.rowptr.get(), n,
                                                                                 T.cnt.get(), nullptr, nullptr, nullptr);
    B200_CUDA(cudaGetLastError());
    count_launch();
    T.scan_counts(n, 0);
    long long c = 0;
    B200_CUDA(cudaMemcpy(&c, T.rowptr_new.get() + n, sizeof(long long), cudaMemcpyDeviceToHost));
    *nnz = c;
  });
}

int b200_slim_tree_csr(b200_slim_t h, int64_t* indptr, int32_t* indices, float* data) {
  return guarded([&] {
    B200_REQUIRE(h && indptr && h->tree, "b200_slim_tree_csr: not a tree-mode handle");
    const int n = h->p.n_items;
    TreeStore& T = h->ts;
    const int grid = std::min<int>(div_up(n, 8), sm_count() * 16);
    B200_CUDA(cudaDeviceSynchronize());
    slim_tree_export_kernel<<<grid, 256>>>(T.key.get(), T.val.get(), T.rowptr.get(), n, T.cnt.get(), nullptr, nullptr, nullptr);
    B200_CUDA(cudaGetLastError());
    T.scan_counts(n, 0);
    long long c = 0;
    B200_CUDA(cudaMemcpy(&c, T.rowptr_new.get() + n, sizeof(long long), cudaMemcpyDeviceToHost));
    B200_REQUIRE(c == 0 || (indices && data), "b200_slim_tree_csr: NULL argument");
    DevBuf<int> d_idx((size_t)std::max(c, 1ll));
    DevBuf<float> d_val((size_t)std::max(c, 1ll));
    slim_tree_export_kernel<<<grid, 256>>>(T.key.get(), T.val.get(), T.rowptr.get(), n, nullptr, T.rowptr_new.get(), d_idx.get(),
                                           d_val.get());
    B200_CUDA(cudaGetLastError());
    count_launch(3);
    B200_CUDA(cudaMemcpy(indptr, T.rowptr_new.get(), sizeof(long long) * ((size_t)n + 1), cudaMemcpyDeviceToHost));
    if (c) {
      B200_CUDA(cudaMemcpy(indices, d_idx.get(), sizeof(int) * (size_t)c, cudaMemcpyDeviceToHost));
      B200_CUDA(cudaMemcpy(data, d_val.get(), sizeof(float) * (size_t)c, cudaMemcpyDeviceToHost));
    }
  });
}

int b200_slim_tree_cells(b200_slim_t h, int64_t* cells) {
  return guarded([&] {
    B200_REQUIRE(h && cells && h->tree, "b200_slim_tree_cells: not a tree-mode handle");
    *cells = h->ts.m;
  });
}

int b200_slim_get_samples(b200_slim_t h, int32_t* u, int32_t* i, int32_t* j) {
  return guarded([&] {
    B200_REQUIRE(h && u && i && j, "b200_slim_get_samples: NULL argument");
    h->ss.copy_out(u, i, j, nullptr);
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
    if (!h->tree) ensure_dense_S(h, 0);
    // the epoch kernels run on the caller's stream (possibly a non-blocking one) and need not have finished: this entry
    // point has no stream argument, so it waits for the whole device before it reads S on the default stream
    B200_CUDA(cudaDeviceSynchronize());
    if (h->tree) {  // the cells scattered into the zeroed view
      B200_CUDA(cudaMemset(dst, 0, cells * sizeof(float)));
      if (h->ts.m) slim_tree_scatter_kernel<<<div_up(h->ts.m, 256), 256>>>(h->ts.key.get(), h->ts.val.get(), h->ts.m, n, dst);
    } else {
      slim_full_kernel<<<div_up((long long)cells, 256), 256>>>(h->p.S, n, h->p.symmetric, dst);
    }
    B200_CUDA(cudaGetLastError());
    count_launch();
    if (h_out) B200_CUDA(cudaMemcpy(h_out, dst, cells * sizeof(float), cudaMemcpyDeviceToHost));
    else B200_CUDA(cudaDeviceSynchronize());
  });
}

int b200_slim_last_epoch_ms(b200_slim_t h, float* ms) {
  return guarded([&] {
    B200_REQUIRE(h && ms && h->timer.timed, "b200_slim_last_epoch_ms: no epoch run yet");
    h->timer.elapsed(ms);
  });
}

}  // extern "C"
