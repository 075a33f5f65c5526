// K1: sparse column-column similarity with exact top-K selection, sm_90a.
//
// Replaces Base/Similarity/Cython/Compute_Similarity_Cython.pyx:327-408 (computeItemSimilarities, the
// Gustavson row-gather into an n_columns accumulator) and :467-568 (normalise, top-K, emit).
//
// Design (DESIGN.md "K1").  At create time the columns are RENUMBERED by ascending norm term B_j (ties by
// original index), the CSR rows re-sorted in the new numbering and the CSC built from them.  One persistent
// CTA per SM pulls target columns from an atomic counter.  For a target column i the CTA stages i's CSC
// entries (user, x_ui * w_u) in shared memory, then -- one window of the neighbour axis at a time -- every
// warp streams whole CSR row segments of those users with coalesced loads and scatter-adds x_ui*x_uj into a
// shared-memory accumulator covering the window (fp32 CAS-add, or a native integer ATOMS add when every
// stored value is 1).  Rows are sorted, so the part of a row inside window w is a contiguous range whose
// bounds are precomputed (`split`).  Selection per window:
//   bootstrap  (first window only) a histogram of per-cell similarity LOWER bounds gives a floor `thr` of
//              the K-th best similarity;
//   scan       cells whose dot product is below a per-tile threshold (the analytic inverse of the
//              similarity formula at `thr`, using the norm range of the 4096-cell tile -- tight because
//              norms are monotone in the new numbering) are zeroed unread; the rest are appended as
//              provisional (dot, j) records;
//   evaluate   all records gather (B_j, original index) together, become exact 64-bit keys
//              (similarity bits << 32 | ~original index, so ties resolve to the ascending index) or drop out;
//   select     a range-normalised 2048-bin radix select keeps the K best whenever the buffer runs half full
//              and after the last window.
// Bytes per gathered entry: 8 (index + value) or 4 (binary path).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <stdlib.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "select.cuh"

namespace b200 {
namespace sim {

typedef unsigned long long u64;

constexpr int THREADS = 1024;
constexpr int NWARPS = THREADS / 32;
constexpr int STAGE_INTS = 3072; // staging area: per staged user one value + sp_stride row-segment bounds
constexpr int SPMAX = 5;        // staged split columns per user (all windows at once when n_win + 1 <= SPMAX)
constexpr int HBINS = 4096;     // bootstrap histogram bins (aliases the candidate buffer)
constexpr int SBINS = 2048;     // select histogram bins (aliases the staging area)
#ifndef B200_SELT
#define B200_SELT 256
#endif
constexpr int SELT = B200_SELT;  // threads that run the select
#ifndef B200_UB
#define B200_UB 2
#endif
constexpr int UB = B200_UB;      // 128-bit loads in flight per lane
constexpr int MAXTILES = 16;
#define B200_MAX_PEERS 8  // output tables one launch can write: the local one + up to 7 peers of an 8-GPU box

enum Formula { F_PROD = 0, F_NONORM = 1, F_JACCARD = 2, F_DICE = 3, F_TVERSKY = 4, F_SCALE = 5, F_EUCLID = 6 };

struct KParams {
  int n_cols, K, n_win, win, cap, cap_alloc;  // cap <= cap_alloc (a smaller logical cap is a test hook)
  int acc_cells;     // 4-byte accumulator words allocated (>= SBINS: the cleared window doubles as select scratch)
  int lpu_log2;      // lanes that share one row segment in the accumulate phase (2^lpu_log2, 2..32)
  float se;          // shrink + 1e-6
  float shrink_div;  // shrink if != 0 else 1
  float ta, tb;
  const int* __restrict__ csr_ptr;
  const int2* __restrict__ csr_ent;  // (new column index, value bits), rows sorted by new index
  const int* __restrict__ csr_idx;   // binary path: new column indices only
  const int* __restrict__ split;
  const int* __restrict__ csc_ptr;   // by new column index
  const int2* __restrict__ csc_ent;
  const int* __restrict__ csc_idx;
  const float* __restrict__ A;       // by new column index
  const int2* __restrict__ BN;       // by new column index: (B_j bits, original index); B ascending
  const float* __restrict__ tileB;   // [n_win][MAXTILES + 1]: B at the tile boundaries of every window
  const int* __restrict__ old2new;
  int col_begin, n_range;            // original numbering
  const int* __restrict__ order;     // processing order of local columns (descending work), or nullptr
  int* counter;
  // output tables [columns of the range, K] idx / val and [columns] cnt: n_out copies -- the local one first, then (multi-GPU,
  // b200_sim_compute_peers_device) the same rows of every peer's table, written straight over NVLink by the CTA that
  // finished the column, so that no collective follows the kernel
  int n_out;
  int* o_idx[B200_MAX_PEERS];
  float* o_val[B200_MAX_PEERS];
  int* o_cnt[B200_MAX_PEERS];
  int signed_data;
  // euclidean (Compute_Similarity_Euclidean.py): distance -> similarity mode 0 exp / 1 lin / 2 log, normalize,
  // divisor of normalize_avg_row (n_rows, or 1), shrink as a float, and whether stored values can be negative
  int eu_mode, eu_norm, eu_signed;
  float eu_div, eu_shrink;
  float* dense_out;  // dense mode (TopK == 0 / full Gram): [n_range, n_cols] row-major, out[target - col_begin, neighbour]
  // K1-D (sim_k1d.cuh): 4-bit counter words, key-buffer slots, norm tiles and their bounds, the packed (doubled when the
  // pair path can use it) row layout with the CSC-side (first chunk, chunks) list and the increments every column's rows
  // produce, the work items of the launch (new column, local column, csc begin, csc end), the list + counter that receive
  // the columns to redo, and a test hook (every n-th column is handed back)
  int bm_words, cap_d, fail_every, ntile;
  const float* __restrict__ tbnd;
  const int4* __restrict__ csr_idx1;
  const int2* __restrict__ csc_seg;
  const int* __restrict__ col_adds;
  const int4* __restrict__ worklist;
  int* redo;
  int* fail;
  const int* n_range_dev;  // window kernel / K1-D kernel: the number of columns to process is read from here when set
  // K1-D pair path (sim_k1d.cuh): per CSC entry the column's window in the user's doubled row, the work items in
  // window-work order; the own lists (column i's count >= 3 cells (j << 4 | count), j in i's window, one contiguous run per column:
  // start and length by column), their capacity and fill; the loose list of (i << 32 | j << 4 | count) cells that did not fit
  // a column's stage, its capacity and fill; the per-column mirror counts (deg) and offsets and the mirror lists built from
  // them ((i << 4 | count) in the list of j) through the exchange's destination tiles (2^tile_log2 columns each, fill
  // counters, bucket buffer); the flag that sends the whole call down the K1-D kernel, and the columns that the
  // select kernel hands to the K1-D kernel
  const int2* __restrict__ csc_win;
  const int4* __restrict__ worklist_up;
  unsigned* own;
  int* own_off;
  int* own_n;  // | OWN_SPILLED when the column's cells overflowed its stage
  u64* n_own;
  long long pair_cap;
  u64* loose;
  u64* n_loose;
  long long loose_cap;
  int* deg;
  const int* __restrict__ mir_off;
  unsigned* mir;
  int tile_log2;
  int* tile_fill;
  u64* bucket;
  int* pair_fail;
  int sel_cap;  // the longest list the select kernel decides (its per-warp key buffer)
  int4* wl_redo;
  int* n_redo;
  float lvl_b1, lvl_b2;  // smallest norm term of the columns with >= 1 / >= 2 users (the neighbours a count-1 / -2 cell can have)
  unsigned long long* prof;  // optional [16] per-phase cycle counters (thread 0 of every CTA), test/bench hook
};

__device__ __forceinline__ void emit_entry(const KParams& p, size_t pos, int idx, float val) {
#pragma unroll 1
  for (int r = 0; r < p.n_out; ++r) { p.o_idx[r][pos] = idx; p.o_val[r][pos] = val; }
}
__device__ __forceinline__ void emit_count(const KParams& p, int row, int n) {
#pragma unroll 1
  for (int r = 0; r < p.n_out; ++r) p.o_cnt[r][row] = n;
}

template <int F>
__host__ __device__ __forceinline__ float sim_value(const KParams& p, float d, float a, float b) {
  if (F == F_PROD) return d / (a * b + p.se);
  if (F == F_NONORM) return d / p.shrink_div;
  if (F == F_JACCARD) return d / (a + b - d + p.se);
  if (F == F_DICE) return d / (a + b + p.se);
  if (F == F_SCALE) return d * a * b;  // P3alpha / RP3beta: dot * (1/deg_i)^alpha * deg_j^-beta
  return d / (d + (a - d) * p.ta + (b - d) * p.tb + p.se);
}

// Euclidean similarity of two columns from their squared distance (Compute_Similarity_Euclidean.py:152-173; fp32
// like the reference's arrays): optional division by the product of the norms where that is non-zero (:152-154) and
// by n_rows (:156-157), square root where positive (:159-160), then 1 / (g(d) + shrink + 1e-9) (:162-169).
__device__ __forceinline__ float euclid_sim(const KParams& p, float d2, float sq_i, float sq_j) {
  float d = d2;
  if (p.eu_norm) {
    const float den = sqrtf(sq_i) * sqrtf(sq_j);
    if (den != 0.f) d = d / den;
  }
  d = d / p.eu_div;
  if (d > 0.f) d = sqrtf(d);
  const float g = p.eu_mode == 0 ? expf(d) : (p.eu_mode == 1 ? d : logf(d + 1.f));
  return 1.f / ((g + p.eu_shrink) + 1e-9f);
}

// Smallest positive dot product whose similarity can reach `t` (>0) for ANY neighbour norm term in
// [b_lo, b_hi]: the analytic inverse of sim_value in d at both ends, widened by 1e-5 so that fp32 rounding
// never excludes a qualifying cell.
template <int F>
__device__ __forceinline__ float dot_threshold(const KParams& p, float t, float a, float b_lo, float b_hi) {
  float r = 3.4e38f;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float b = e ? b_hi : b_lo;
    float v;
    if (F == F_PROD) v = t * (a * b + p.se);
    else if (F == F_NONORM) v = t * p.shrink_div;
    else if (F == F_JACCARD) v = t * (a + b + p.se) / (1.f + t);
    else if (F == F_DICE) v = t * (a + b + p.se);
    else if (F == F_SCALE) v = (a * b > 0.f) ? t / (a * b) : 3.4e38f;
    else {
      const float den = 1.f - t * (1.f - p.ta - p.tb);
      v = den > 1e-6f ? t * (a * p.ta + b * p.tb + p.se) / den : 0.f;
    }
    r = fminf(r, v);
  }
  return r > 0.f ? r * (1.f - 1e-5f) : 0.f;
}

// s such that sim_value(d, a, b) >= d * s for every positive d the data can produce and every b in
// [b_lo, b_hi] (a cheap per-tile lower bound for the bootstrap histogram); 0 when no useful bound exists.
template <int F>
__device__ __forceinline__ float lower_bound_scale(const KParams& p, float a, float b_lo, float b_hi) {
  const float b = fmaxf(b_lo, b_hi);
  float den;
  if (F == F_SCALE) return a * fminf(b_lo, b_hi) * (1.f - 1e-5f);
  if (F == F_PROD) den = a * b + p.se;
  else if (F == F_NONORM) den = p.shrink_div;
  else if (F == F_JACCARD || F == F_DICE) den = a + b + p.se;  // jaccard: the "- d" only raises the value
  else {
    // tversky on set data: d <= a, so d*(1-ta-tb) <= a*max(0, 1-ta-tb)
    if (p.ta < 0.f || p.tb < 0.f) return 0.f;
    den = a * fmaxf(0.f, 1.f - p.ta - p.tb) + a * p.ta + b * p.tb + p.se;
  }
  return den > 0.f ? (1.f - 1e-5f) / den : 0.f;
}

#define PROF_MARK(ph)                                                        \
  do {                                                                      \
    if (p.prof && threadIdx.x == 0) {                                       \
      const long long _t = clock64();                                       \
      atomicAdd(p.prof + (ph), (unsigned long long)(_t - prof_t));          \
      prof_t = _t;                                                          \
    }                                                                       \
  } while (0)
// the same from lane 0 of every warp (kernels that work one column per warp; prof_t per warp)
#define PROF_MARK_WARP(ph)                                                   \
  do {                                                                      \
    if (p.prof && (threadIdx.x & 31) == 0) {                                \
      const long long _t = clock64();                                       \
      atomicAdd(p.prof + (ph), (unsigned long long)(_t - prof_t));          \
      prof_t = _t;                                                          \
    }                                                                       \
  } while (0)

template <bool NEG>
__device__ __forceinline__ unsigned key32_of(float v) {
  return NEG ? ~__float_as_uint(v) : __float_as_uint(v);
}

struct Shared {
  int col;
  int nbuf;
  int overflow;
  int npos, nneg;
  int digit, need, bincnt;
  int b0;
  int cnt;
  unsigned kmin, kmax;
  u64 sel_thr;
  int warp_tot[NWARPS];
  float dthr[MAXTILES];
  float lbs[MAXTILES];
  unsigned k2[MAXTILES];  // packed path: (0x8000 - ceil(dthr)) in both half-words, see half_ge_mask
};

// Bootstrap histogram bins: 6 mantissa bits (1.6% steps) over the exponents 2^-40 .. 2^24; smaller values share
// bin 0 (never used as a floor), larger ones the top bin (whose lower edge is still a valid floor).
constexpr int LB_BASE = (127 - 40) << 6;
__device__ __forceinline__ int lb_bin(const float lb) {
  return min(max((int)(__float_as_uint(lb) >> 17) - LB_BASE, 0), HBINS - 1);
}
__device__ __forceinline__ unsigned lb_bin_floor_bits(const int b) { return ((unsigned)(b + LB_BASE)) << 17; }

// Packed 16-bit counters (all < 0x8000): bit q / bit 16+q of the result is set iff the low / high half-word of
// word q of `v` is >= t, where k2 = (0x8000 - t) * 0x10001 and 1 <= t <= 0x8000 (no carry crosses the half-words).
__device__ __forceinline__ unsigned half_ge_mask(const uint4 v, const unsigned k2) {
  const unsigned M = 0x80008000u;
  return (((v.x + k2) & M) >> 15) | (((v.y + k2) & M) >> 14) | (((v.z + k2) & M) >> 13) | (((v.w + k2) & M) >> 12);
}
__device__ __forceinline__ unsigned half_k2(const float dthr) {
  const unsigned t = dthr <= 1.f ? 1u : (dthr >= 32768.f ? 0x8000u : (unsigned)ceilf(dthr));
  return (0x8000u - t) * 0x10001u;
}

__device__ __forceinline__ void bar_sel() { asm volatile("bar.sync 1, %0;" ::"n"(SELT) : "memory"); }

// exclusive suffix sum over the block: returns sum of v over all threads with a larger thread index
__device__ __forceinline__ int block_suffix_excl(int v, int* warp_tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    int t = __shfl_down_sync(0xffffffffu, incl, off);
    if (lane + off < 32) incl += t;
  }
  if (lane == 0) warp_tot[warp] = incl;
  __syncthreads();
  int above = 0;
  for (int w = warp + 1; w < NWARPS; ++w) above += warp_tot[w];
  __syncthreads();
  return above + incl - v;
}

// Called by threads 0..SELT-1 only (named barrier 1).  buf[0..n) holds distinct keys, some of them 0 (dead
// slots).  Keeps the K largest non-zero keys (all of them if there are at most K) compacted at the front of
// buf, writes the surviving count to sh->cnt and a threshold to sh->sel_thr such that exactly the survivors
// are >= it (0 when nothing was cut).  Radix select over the occupied key range: every level maps the
// still-undecided keys linearly onto SBINS bins (they spread out instead of piling onto one counter), finds
// the bin holding the K-th key and narrows to it; stops as soon as a bin is taken whole.
__device__ void select_group(u64* buf, int n, int K, Shared* sh, int* hist) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int SW = SELT / 32;
  for (int i = tid; i < SBINS; i += SELT) hist[i] = 0;
  if (tid == 0) { sh->kmin = 0xFFFFFFFFu; sh->kmax = 0u; sh->cnt = 0; }
  bar_sel();
  {
    unsigned mn = 0xFFFFFFFFu, mx = 0u;
    int valid = 0;
    for (int q = tid; q < n; q += SELT) {
      const u64 k = buf[q];
      if (k) {
        const unsigned h = (unsigned)(k >> 32);
        mn = min(mn, h);
        mx = max(mx, h);
        ++valid;
      }
    }
    mn = __reduce_min_sync(0xffffffffu, mn);
    mx = __reduce_max_sync(0xffffffffu, mx);
    valid = __reduce_add_sync(0xffffffffu, valid);
    if (lane == 0) { atomicMin(&sh->kmin, mn); atomicMax(&sh->kmax, mx); atomicAdd(&sh->cnt, valid); }
  }
  bar_sel();
  const int valid = sh->cnt;
  u64 thr = 0;
  if (valid > K) {
    u64 base = ((u64)sh->kmin) << 32;
    const u64 top = (((u64)sh->kmax) << 32) | 0xFFFFFFFFull;
    int width = 64 - __clzll((long long)(top - base));  // live keys lie in [base, base + 2^width)
    int need = K;
    while (true) {
      const int shift = max(0, width - 11);
      for (int q = tid; q < n; q += SELT) {
        const u64 k = buf[q];
        const u64 off = k - base;
        if (k >= base && k != 0ull && (width >= 64 || (off >> width) == 0ull)) atomicAdd(&hist[(int)(off >> shift)], 1);
      }
      bar_sel();
      // SBINS / SELT = 16 bins per thread, highest bins in the highest threads
      int c[SBINS / SELT], local = 0;
#pragma unroll
      for (int b = 0; b < SBINS / SELT; ++b) {
        c[b] = hist[tid * (SBINS / SELT) + b];
        hist[tid * (SBINS / SELT) + b] = 0;
        local += c[b];
      }
      int incl = local;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_down_sync(0xffffffffu, incl, off);
        if (lane + off < 32) incl += t;
      }
      if (lane == 0) sh->warp_tot[warp] = incl;
      bar_sel();
      int cum = incl - local;
      for (int w = warp + 1; w < SW; ++w) cum += sh->warp_tot[w];
#pragma unroll
      for (int b = SBINS / SELT - 1; b >= 0; --b) {
        if (cum < need && cum + c[b] >= need) { sh->digit = tid * (SBINS / SELT) + b; sh->need = need - cum; sh->bincnt = c[b]; }
        cum += c[b];
      }
      bar_sel();
      base += ((u64)sh->digit) << shift;
      need = sh->need;
      const int bincnt = sh->bincnt;
      width = shift;
      bar_sel();
      if (bincnt == need || shift == 0) break;
    }
    thr = base;
  }
  // compaction: survivors are gathered into registers (n <= 64 * SELT), then rewritten from the front
  if (tid == 0) sh->cnt = 0;
  u64 keep[16];
  const int rounds = (n + SELT - 1) / SELT;
  for (int r0 = 0; r0 < rounds; r0 += 16) {
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int i = (r0 + q) * SELT + tid;
      const u64 k = (r0 + q < rounds && i < n) ? buf[i] : 0ull;
      keep[q] = (k != 0ull && k >= thr) ? k : 0ull;
    }
    bar_sel();
    // positions written are always < positions still unread (count of survivors so far <= entries consumed)
#pragma unroll
    for (int q = 0; q < 16; ++q)
      if (keep[q]) buf[atomicAdd(&sh->cnt, 1)] = keep[q];
    bar_sel();
  }
  if (tid == 0) sh->sel_thr = thr;
}

// block-wide wrapper: threads >= SELT wait
__device__ __forceinline__ u64 block_select(u64* buf, int n, int K, Shared* sh, int* hist, int* n_out) {
  __syncthreads();
  if (threadIdx.x < SELT) select_group(buf, n, K, sh, hist);
  __syncthreads();
  *n_out = sh->cnt;
  return sh->sel_thr;
}

// cells of one 16-byte vector of the accumulator window as floats: 4 fp32 / int32 cells, or 8 packed 16-bit counters
template <bool BINARY, bool PACK>
__device__ __forceinline__ bool load_cells(const void* acc, int iv, float* d) {
  if (PACK) {
    const int4 v = reinterpret_cast<const int4*>(acc)[iv];
    if ((v.x | v.y | v.z | v.w) == 0) return false;
    d[0] = (float)(v.x & 0xFFFF); d[1] = (float)((unsigned)v.x >> 16); d[2] = (float)(v.y & 0xFFFF); d[3] = (float)((unsigned)v.y >> 16);
    d[4] = (float)(v.z & 0xFFFF); d[5] = (float)((unsigned)v.z >> 16); d[6] = (float)(v.w & 0xFFFF); d[7] = (float)((unsigned)v.w >> 16);
    return true;
  } else if (BINARY) {
    const int4 v = reinterpret_cast<const int4*>(acc)[iv];
    if ((v.x | v.y | v.z | v.w) == 0) return false;
    d[0] = (float)v.x; d[1] = (float)v.y; d[2] = (float)v.z; d[3] = (float)v.w;
    return true;
  } else {
    const float4 v = reinterpret_cast<const float4*>(acc)[iv];
    if (v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) return false;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    return true;
  }
}

template <bool BINARY, bool PACK>
__device__ __forceinline__ void store_cells(void* acc, int iv, const float* k) {
  if (PACK) {
    reinterpret_cast<int4*>(acc)[iv] = make_int4((int)k[0] | ((int)k[1] << 16), (int)k[2] | ((int)k[3] << 16),
                                                 (int)k[4] | ((int)k[5] << 16), (int)k[6] | ((int)k[7] << 16));
  } else if (BINARY) {
    reinterpret_cast<int4*>(acc)[iv] = make_int4((int)k[0], (int)k[1], (int)k[2], (int)k[3]);
  } else {
    reinterpret_cast<float4*>(acc)[iv] = make_float4(k[0], k[1], k[2], k[3]);
  }
}

template <int F, bool BINARY, bool PACK, bool NEG>
__device__ void process_column(const KParams& p, int col, int target, int out_base, unsigned char* smem_raw,
                               Shared* sh, const float* s_tileB, int* n_emitted) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* accf = reinterpret_cast<float*>(smem_raw);
  int* acci = reinterpret_cast<int*>(smem_raw);
  u64* buf = reinterpret_cast<u64*>(smem_raw + (size_t)p.acc_cells * 4);
  int* hist = reinterpret_cast<int*>(buf);
  int* stage = reinterpret_cast<int*>(buf + p.cap_alloc);
  int* shist_stage = stage;  // select scratch while the window still holds cells (SBINS <= STAGE_INTS)
  bool staged_valid = false;

  const int cs = p.csc_ptr[col], ce = p.csc_ptr[col + 1];
  const float Ai = p.A[col];
  long long prof_t = p.prof ? clock64() : 0;
  u64 thr = 0;
  int nbuf = 0;
  if (tid == 0) { sh->nbuf = 0; if (!NEG) { sh->npos = 0; sh->nneg = 0; } }

  // all window bounds of a user are staged at once when they fit (one trip to memory per column instead of
  // one per window); columns longer than a chunk, or many windows, restage per (window, chunk)
  const bool all_splits = (p.n_win + 1 <= SPMAX) && (ce - cs <= STAGE_INTS / (p.n_win + 2));
  const int sp_stride = all_splits ? (p.n_win + 1) : 2;
  const int colchunk = STAGE_INTS / (1 + sp_stride);  // users staged per chunk
  float* sm_x = reinterpret_cast<float*>(stage);
  int* sm_sp = stage + colchunk;
  const int lpu = 1 << p.lpu_log2, upw = 32 >> p.lpu_log2;  // lanes per user, users per warp slot
  const int sub = lane & (lpu - 1), uslot = lane >> p.lpu_log2;
  __syncthreads();

  if (F == F_EUCLID) {
    // Every column -- co-rated or not -- has a finite distance to the target, so the candidates are ALL cells.  A floor
    // of the target-th best similarity comes from the norms alone: for any neighbour j the squared distance is at most
    // sq_i + sq_j (non-negative data: dot >= 0) or (|i| + |j|)^2 (signed data), so the target-th best of those bounds
    // over ANY set of cells is a valid floor.  The set: the columns next to the target in norm order (normalize: the
    // zero-dot distance |i|/|j| + |j|/|i| is smallest around |j| = |i|) or the smallest norms (plain distance).
    const int lo = p.eu_norm ? max(0, col - target) : 0;
    const int hi = p.eu_norm ? min(p.n_cols, col + target + 1) : min(p.n_cols, target + 1);
    for (int t = lo + tid; t < hi; t += THREADS) {
      u64 key = 0ull;
      if (t != col) {
        const int2 bn = __ldg(p.BN + t);
        const float b = __int_as_float(bn.x);
        const float dmax2 = p.eu_signed ? (Ai + b) + 2.f * sqrtf(Ai) * sqrtf(b) : (Ai + b);
        const float sv = euclid_sim(p, dmax2, Ai, b);
        if (sv > 0.f) key = (((u64)__float_as_uint(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn.y);
      }
      buf[t - lo] = key;
    }
    int kept;
    const u64 t0 = block_select(buf, hi - lo, target, sh, acci, &kept);  // the window is all zero here
    if (t0) thr = ((u64)__float_as_uint(__uint_as_float((unsigned)(t0 >> 32)) * (1.f - 1e-5f))) << 32;
    if (tid == 0) sh->nbuf = 0;
    __syncthreads();
  }

  for (int w = 0; w < p.n_win; ++w) {
    const int win_lo = w * p.win;
    const int win_n = min(p.win, p.n_cols - win_lo);
    constexpr int CPV = PACK ? 8 : 4;  // cells per 16-byte vector
    const int winv = (win_n + CPV - 1) / CPV;
    const int ntiles = (winv + THREADS - 1) / THREADS;
    const float* tB = s_tileB + w * (MAXTILES + 1);
    int* accw_i = acci - win_lo;
    float* accw_f = accf - win_lo;
    unsigned* accw_u = reinterpret_cast<unsigned*>(acci) - (win_lo >> 1);  // packed: cell j lives in word j >> 1

    // ---------------- accumulate: acc[j - win_lo] += x_ui * x_uj over users u of column `col`
    for (int k0 = cs; k0 < ce; k0 += colchunk) {
      const int n = min(colchunk, ce - k0);
      if (!all_splits || !staged_valid) {
        staged_valid = true;
        __syncthreads();
        for (int t = tid; t < n; t += THREADS) {
          int u;
          if (BINARY) {
            u = p.csc_idx[k0 + t];
          } else {
            const int2 e = p.csc_ent[k0 + t];
            u = e.x;
            sm_x[t] = __int_as_float(e.y);
          }
          if (p.n_win == 1 && !BINARY) {
            sm_sp[t * 2] = p.csr_ptr[u];
            sm_sp[t * 2 + 1] = p.csr_ptr[u + 1];
          } else if (all_splits) {
            const int* sp = p.split + (size_t)u * (p.n_win + 1);
            for (int q = 0; q <= p.n_win; ++q) sm_sp[t * sp_stride + q] = sp[q];
          } else {
            const int* sp = p.split + (size_t)u * (p.n_win + 1) + w;
            sm_sp[t * 2] = sp[0];
            sm_sp[t * 2 + 1] = sp[1];
          }
        }
        __syncthreads();
      }
      PROF_MARK(0);
      const int spo = all_splits ? w : 0;
      for (int t0 = warp * upw; t0 < n; t0 += NWARPS * upw * UB) {
        int s[UB], e[UB], a0[UB];
        float x[UB];
        int mych = 0;
#pragma unroll
        for (int k = 0; k < UB; ++k) {
          const int t = t0 + k * NWARPS * upw + uslot;
          if (t < n) {
            s[k] = sm_sp[t * sp_stride + spo];
            e[k] = sm_sp[t * sp_stride + spo + 1];
            x[k] = BINARY ? 1.f : sm_x[t];
          } else {
            s[k] = 0; e[k] = 0; x[k] = 0.f;
          }
          // 16-byte chunks: 4 indices (binary; every (row, window) segment is 16-byte aligned and padded with a
          // dummy cell index, so there are no partial chunks) or 2 (index, value) pairs
          a0[k] = BINARY ? s[k] : (s[k] & ~1);
          mych = max(mych, BINARY ? ((e[k] - a0[k]) >> 2) : ((e[k] - a0[k] + 1) >> 1));
        }
        const int maxch = __reduce_max_sync(0xffffffffu, mych);
        for (int c0 = 0; c0 < maxch; c0 += lpu) {
          const int ch = c0 + sub;
          int4 v[UB];
#pragma unroll
          for (int k = 0; k < UB; ++k) {
            const int g = a0[k] + ch * (BINARY ? 4 : 2);
            v[k] = make_int4(-1, -1, -1, -1);
            if (g < e[k]) v[k] = BINARY ? __ldg(reinterpret_cast<const int4*>(p.csr_idx + g))
                                        : __ldg(reinterpret_cast<const int4*>(p.csr_ent + g));
          }
#pragma unroll
          for (int k = 0; k < UB; ++k) {
            const int g = a0[k] + ch * (BINARY ? 4 : 2);
            // the diagonal is accumulated like any other cell and zeroed after the loop
            if (BINARY) {
              if (g < e[k]) {
                const int jj[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  if (PACK) atomicAdd(&accw_u[jj[c] >> 1], (jj[c] & 1) ? 65536u : 1u);
                  else atomicAdd(&accw_i[jj[c]], 1);
                }
              }
            } else {
              if (g >= s[k] && g < e[k]) atomicAdd(&accw_f[v[k].x], x[k] * __int_as_float(v[k].y));
              if (g + 1 >= s[k] && g + 1 < e[k]) atomicAdd(&accw_f[v[k].z], x[k] * __int_as_float(v[k].w));
            }
          }
        }
      }
    }
    __syncthreads();
    if (tid == 0 && col >= win_lo && col < win_lo + win_n) {  // pyx:396
      const int c = col - win_lo;
      if (PACK) acci[c >> 1] &= (c & 1) ? 0x0000FFFF : (int)0xFFFF0000; else acci[c] = 0;
    }
    __syncthreads();
    PROF_MARK(1);
    if (p.dense_out) {
      // dense mode (pyx:510-513): every non-zero cell is normalised and written out, no selection
      float* orow = p.dense_out + (size_t)out_base * p.n_cols;  // out_base = local target index here
      for (int c = tid; c < win_n; c += THREADS) {
        const float d = PACK ? (float)(((unsigned)acci[c >> 1] >> ((c & 1) * 16)) & 0xFFFFu) : (BINARY ? (float)acci[c] : accf[c]);
        if (d != 0.f) {
          const int2 bn = __ldg(p.BN + win_lo + c);
          orow[bn.y] = sim_value<F>(p, d, Ai, __int_as_float(bn.x));
        }
      }
      __syncthreads();
      for (int iv = tid; iv < winv; iv += THREADS) reinterpret_cast<int4*>(acci)[iv] = make_int4(0, 0, 0, 0);
      __syncthreads();
      continue;
    }

    if (F == F_EUCLID) {
      // every cell of the window is evaluated exactly, 1024 at a time; the buffer is pruned to the best `target`
      // (raising thr to an exact key) whenever the next chunk might not fit, so nothing ever overflows
      int ub = sh->nbuf;  // block-uniform upper bound of sh->nbuf (every chunk pushes at most THREADS keys)
      __syncthreads();
      for (int c0 = 0; c0 < win_n; c0 += THREADS) {
        if (ub + THREADS > p.cap) {
          ub = sh->nbuf;      // exact: the pushes of the previous chunk ended at its barrier
          __syncthreads();    // nobody pushes again before everybody has read it
          if (ub + THREADS > p.cap) {
            int kept;
            staged_valid = false;  // the staging area is the select scratch while cells remain in the window
            thr = max(thr, block_select(buf, ub, target, sh, shist_stage, &kept));
            if (tid == 0) sh->nbuf = kept;
            ub = kept;
            __syncthreads();
          }
        }
        ub += THREADS;
        const int c = c0 + tid;
        if (c < win_n && win_lo + c != col) {
          const float d = PACK ? (float)(((unsigned)acci[c >> 1] >> ((c & 1) * 16)) & 0xFFFFu) : (BINARY ? (float)acci[c] : accf[c]);
          const int2 bn = __ldg(p.BN + win_lo + c);
          const float b = __int_as_float(bn.x);
          const float sv = euclid_sim(p, (b + Ai) - 2.f * d, Ai, b);
          const u64 key = (((u64)__float_as_uint(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn.y);
          if (sv > 0.f && key >= thr) buf[atomicAdd(&sh->nbuf, 1)] = key;
        }
        __syncthreads();
      }
      for (int iv = tid; iv < winv; iv += THREADS) reinterpret_cast<int4*>(acci)[iv] = make_int4(0, 0, 0, 0);
      __syncthreads();
      nbuf = sh->nbuf;
      if (w == p.n_win - 1) {
        int kept;
        thr = max(thr, block_select(buf, nbuf, target, sh, acci, &kept));
        if (tid == 0) sh->nbuf = kept;
        nbuf = kept;
        __syncthreads();
      }
      PROF_MARK(3);
      continue;
    }

    nbuf = sh->nbuf;
    // ---------------- bootstrap: floor of the target-th best similarity from per-cell lower bounds
    if (!NEG && thr == 0 && nbuf == 0 && win_n > 2 * target) {
      for (int i = tid; i < HBINS; i += THREADS) hist[i] = 0;
      if (tid == 0) sh->b0 = -1;
      if (tid < ntiles) sh->lbs[tid] = lower_bound_scale<F>(p, Ai, tB[tid], tB[tid + 1]);
      __syncthreads();
      if (PACK) {
        // every lane of a warp is in the same tile in the same iteration, so cells with a count of 1 or 2 (the bulk)
        // land in two bins: count them with half-word compares and add once per warp; counts >= 3 go one by one
        for (int iv0 = warp * 32; iv0 < winv; iv0 += THREADS) {
          const int iv = iv0 + lane;
          const float sc = sh->lbs[iv0 / THREADS];
          uint4 v = make_uint4(0u, 0u, 0u, 0u);
          if (iv < winv) v = reinterpret_cast<const uint4*>(acci)[iv];
          const int n1 = __popc(half_ge_mask(v, 0x7FFF7FFFu)), n2 = __popc(half_ge_mask(v, 0x7FFE7FFEu));
          unsigned m3 = half_ge_mask(v, 0x7FFD7FFDu);
          const int n3 = __popc(m3);
          while (m3) {
            const int b = __ffs(m3) - 1;
            m3 &= m3 - 1;
            const int q = b & 3;
            const unsigned wq = q == 0 ? v.x : (q == 1 ? v.y : (q == 2 ? v.z : v.w));
            const float lb = (float)((b >> 4) ? (wq >> 16) : (wq & 0xFFFFu)) * sc;
            if (lb > 0.f) atomicAdd(&hist[lb_bin(lb)], 1);
          }
          const int c1 = __reduce_add_sync(0xffffffffu, n1 - n2), c2 = __reduce_add_sync(0xffffffffu, n2 - n3);
          if (lane == 0 && sc > 0.f) {
            if (c1) atomicAdd(&hist[lb_bin(sc)], c1);
            if (c2) atomicAdd(&hist[lb_bin(2.f * sc)], c2);
          }
        }
      } else {
        for (int iv = tid; iv < winv; iv += THREADS) {
          const float sc = sh->lbs[iv / THREADS];
          float d[CPV];
          if (!load_cells<BINARY, PACK>(acci, iv, d)) continue;
#pragma unroll
          for (int c = 0; c < CPV; ++c) {
            const float lb = d[c] * sc;
            if (lb > 0.f) atomicAdd(&hist[lb_bin(lb)], 1);
          }
        }
      }
      __syncthreads();
      int hh[HBINS / THREADS], local = 0;
#pragma unroll
      for (int b = 0; b < HBINS / THREADS; ++b) { hh[b] = hist[tid * (HBINS / THREADS) + b]; local += hh[b]; }
      int cum = block_suffix_excl(local, sh->warp_tot);
#pragma unroll
      for (int b = HBINS / THREADS - 1; b >= 0; --b) {
        if (cum < target && cum + hh[b] >= target) sh->b0 = tid * (HBINS / THREADS) + b;
        cum += hh[b];
      }
      __syncthreads();
      const int b0 = sh->b0;
      if (b0 > 0) thr = ((u64)lb_bin_floor_bits(b0)) << 32;
      __syncthreads();  // hist (aliasing buf) fully consumed before candidates are pushed
    }
    PROF_MARK(2);

    // ---------------- scan + clear / evaluate, see the header comment.  A cell that finds the buffer full
    // stays in place; the buffer is then pruned to the best `target` and the rescan picks the leftovers up.
    bool first = true;
    while (true) {
      const int nbuf_old = sh->nbuf;
      __syncthreads();
      if (tid == 0) sh->overflow = 0;
      if (tid < ntiles) {
        const float dt = (!NEG && thr) ? dot_threshold<F>(p, __uint_as_float((unsigned)(thr >> 32)), Ai, tB[tid], tB[tid + 1]) : 0.f;
        sh->dthr[tid] = dt;
        if (PACK) sh->k2[tid] = half_k2(dt);
      }
      int cpos = 0, cneg = 0;
      const bool count_signs = !NEG && first && p.signed_data;
      __syncthreads();
      for (int iv = tid; iv < winv; iv += THREADS) {
        const float dthr = sh->dthr[iv / THREADS];
        if (PACK && !NEG) {
          // counts are non-negative integers: d >= dthr <=> d >= ceil(dthr), tested on all 8 half-words at once; the
          // vector is cleared and only the (few) passing cells are looked at one by one
          const uint4 v = reinterpret_cast<const uint4*>(acci)[iv];
          unsigned m = half_ge_mask(v, sh->k2[iv / THREADS]);
          reinterpret_cast<int4*>(acci)[iv] = make_int4(0, 0, 0, 0);
          while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const int q = b & 3, hf = b >> 4;
            const unsigned wq = q == 0 ? v.x : (q == 1 ? v.y : (q == 2 ? v.z : v.w));
            const unsigned cntv = hf ? (wq >> 16) : (wq & 0xFFFFu);
            const int pos = atomicAdd(&sh->nbuf, 1);
            if (pos < p.cap)
              buf[pos] = (((u64)__float_as_uint((float)cntv)) << 32) | (u64)(unsigned)(win_lo + iv * CPV + 2 * q + hf);
            else {  // stays in place for the rescan
              sh->overflow = 1;
              reinterpret_cast<unsigned short*>(acci)[iv * CPV + 2 * q + hf] = (unsigned short)cntv;
            }
          }
          continue;
        }
        float d[CPV];
        if (!load_cells<BINARY, PACK>(acci, iv, d)) continue;
        if (count_signs) {
#pragma unroll
          for (int c = 0; c < CPV; ++c) {
            // the sign of the similarity, not of the dot product: the scaled product is 0 where A_i or B_j is 0, and such
            // a cell is one of the zeros that outrank the negatives (every other formula keeps the sign of d)
            float s = d[c];
            if (F == F_SCALE && s != 0.f) s = sim_value<F>(p, s, Ai, __int_as_float(__ldg(p.BN + win_lo + iv * CPV + c).x));
            cpos += s > 0.f; cneg += s < 0.f;
          }
        }
        float keepv[CPV];
        float dmax = NEG ? -d[0] : d[0];
#pragma unroll
        for (int c = 0; c < CPV; ++c) { keepv[c] = 0.f; dmax = fmaxf(dmax, NEG ? -d[c] : d[c]); }
        if (dmax > 0.f && dmax >= dthr) {
#pragma unroll
          for (int c = 0; c < CPV; ++c) {
            const float dd = d[c];
            if (NEG ? (dd < 0.f) : (dd > 0.f && dd >= dthr)) {
              const int pos = atomicAdd(&sh->nbuf, 1);
              if (pos < p.cap)
                buf[pos] = (((u64)__float_as_uint(dd)) << 32) | (u64)(unsigned)(win_lo + iv * CPV + c);
              else { sh->overflow = 1; keepv[c] = dd; }
            }
          }
        }
        store_cells<BINARY, PACK>(acci, iv, keepv);
      }
      if (count_signs) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          cpos += __shfl_xor_sync(0xffffffffu, cpos, off);
          cneg += __shfl_xor_sync(0xffffffffu, cneg, off);
        }
        if (lane == 0) { if (cpos) atomicAdd(&sh->npos, cpos); if (cneg) atomicAdd(&sh->nneg, cneg); }
      }
      first = false;
      __syncthreads();
      PROF_MARK(3);
      const int n_end = min(sh->nbuf, p.cap);
      const bool overflow = sh->overflow != 0;
      // evaluate in place: provisional (dot, j) -> exact key, or 0 (dead slot, dropped by the next select)
      for (int e = nbuf_old + tid; e < n_end; e += THREADS) {
        const u64 rec = buf[e];
        const int j = (int)(unsigned)rec;
        const float dd = __uint_as_float((unsigned)(rec >> 32));
        const int2 bn = __ldg(p.BN + j);
        const float sv = sim_value<F>(p, dd, Ai, __int_as_float(bn.x));
        const u64 key = (((u64)key32_of<NEG>(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn.y);
        buf[e] = (key >= thr && (NEG ? (sv < 0.f) : (sv > 0.f))) ? key : 0ull;
      }
      nbuf = n_end;
      __syncthreads();
      if (tid == 0) sh->nbuf = nbuf;
      PROF_MARK(4);
      if (!overflow) break;
      int kept;
      staged_valid = false;  // the staging area is the only scratch left while cells remain in the window
      thr = max(thr, block_select(buf, nbuf, target, sh, shist_stage, &kept));
      if (tid == 0) sh->nbuf = kept;
      __syncthreads();
    }
    __syncthreads();
    nbuf = sh->nbuf;
    if (nbuf > p.cap / 2 || w == p.n_win - 1) {
      int kept;  // the window is all zero here and select leaves its scratch zeroed
      thr = max(thr, block_select(buf, nbuf, target, sh, acci, &kept));
      if (tid == 0) sh->nbuf = kept;
      nbuf = kept;
      __syncthreads();
    }
    PROF_MARK(5);
  }

  // ---------------- emit (keys carry the ORIGINAL neighbour index; the last select left no dead slots)
  for (int t = tid; t < nbuf; t += THREADS) {
    const u64 k = buf[t];
    const unsigned hi = (unsigned)(k >> 32);
    emit_entry(p, (size_t)out_base + t, (int)(0xFFFFFFFFu - (unsigned)k), __uint_as_float(NEG ? ~hi : hi));
  }
  *n_emitted = nbuf;
  __syncthreads();
  PROF_MARK(6);
}

template <int F, bool BINARY, bool PACK>
__global__ void __launch_bounds__(THREADS, 1) sim_topk_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ Shared sh;
  const int tid = threadIdx.x;
  // layout: [acc acc_cells*4][buf cap_alloc*8][stage STAGE_INTS*4][tileB n_win*(MAXTILES+1)*4]
  float* s_tileB = reinterpret_cast<float*>(smem_raw + (size_t)p.acc_cells * 4 + (size_t)p.cap_alloc * 8 +
                                            (size_t)STAGE_INTS * 4);
  {
    const int4 z = make_int4(0, 0, 0, 0);
    for (int i4 = tid; i4 < (p.acc_cells >> 2); i4 += THREADS) reinterpret_cast<int4*>(smem_raw)[i4] = z;
    for (int i = tid; i < p.n_win * (MAXTILES + 1); i += THREADS) s_tileB[i] = p.tileB[i];
  }
  __syncthreads();
  const int n_range = p.n_range_dev ? *p.n_range_dev : p.n_range;
  while (true) {
    if (tid == 0) sh.col = atomicAdd(p.counter, 1);
    __syncthreads();
    const int c = sh.col;
    if (c >= n_range) break;
    const int lc = p.order ? p.order[c] : c;
    const int col = p.old2new[p.col_begin + lc];  // new numbering
    const int out_base_row = lc;
    int n_out = 0;
    if (p.dense_out) {
      process_column<F, BINARY, PACK, false>(p, col, p.K, out_base_row, smem_raw, &sh, s_tileB, &n_out);
      __syncthreads();
      continue;
    }
    process_column<F, BINARY, PACK, false>(p, col, p.K, out_base_row * p.K, smem_raw, &sh, s_tileB, &n_out);
    if (p.signed_data && n_out < p.K) {
      // zeros outrank negatives (Compute_Similarity_Python.py:335-345): negatives are only emitted when the
      // positives plus the implicit zeros (every column without a non-zero similarity, the diagonal
      // included) do not fill K slots.
      const int npos = sh.npos, nneg = sh.nneg;
      const int nzero = p.n_cols - npos - nneg;
      const int m = p.K - n_out - nzero;
      __syncthreads();
      if (m > 0 && nneg > 0) {
        int n_neg_out = 0;
        process_column<F, BINARY, PACK, true>(p, col, m, out_base_row * p.K + n_out, smem_raw, &sh, s_tileB, &n_neg_out);
        n_out += n_neg_out;
      }
    }
    for (int t = n_out + tid; t < p.K; t += THREADS) {
      emit_entry(p, (size_t)out_base_row * p.K + t, -1, 0.f);
    }
    if (tid == 0) emit_count(p, out_base_row, n_out);
    __syncthreads();
  }
}

// B at the tile boundaries of every window: tileB[w][t] = B[min(w*win + t*tile, last column of window w)], tile = cells per block-wide scan step
__global__ void tile_bounds_kernel(const int2* __restrict__ BN, int n_cols, int n_win, int win, int tile, float* tileB) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_win * (MAXTILES + 1)) return;
  const int w = g / (MAXTILES + 1), t = g % (MAXTILES + 1);
  const int win_lo = w * win, win_n = min(win, n_cols - win_lo);
  const int j = min(win_lo + t * tile, win_lo + win_n - 1);
  tileB[g] = __int_as_float(BN[j].x);
}

// ------------------------------------------------------------------------------------------------------
// host helpers of the launch set-up, shared with sim_k1d.cuh
// ------------------------------------------------------------------------------------------------------
typedef void (*sim_kernel_t)(const KParams);

// Calls fn(std::integral_constant<int, F>{}) for the formula F among Fs that equals f, so that fn can name the kernel
// instance that serves f.  The last of Fs also serves every formula not listed.
template <int F, int... Fs, class Fn>
decltype(auto) with_formula(int f, Fn&& fn) {
  if constexpr (sizeof...(Fs) == 0) return fn(std::integral_constant<int, F>{});
  else if (f == F) return fn(std::integral_constant<int, F>{});
  else return with_formula<Fs...>(f, fn);
}

// The dynamic shared-memory limit is an attribute of the kernel, shared by every handle with the same formula and counter
// type, each of which launches with a size of its own: raise it to this handle's size, never lower it (a handle built
// later for a smaller catalogue would otherwise break the launches of a larger one still alive).
template <typename Kernel>
void raise_smem_limit(Kernel kernel, size_t bytes) {
  cudaFuncAttributes fa{};
  B200_CUDA(cudaFuncGetAttributes(&fa, kernel));
  if ((size_t)fa.maxDynamicSharedSizeBytes < bytes)
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

#include "sim_k1d.cuh"

// ------------------------------------------------------------------------------------------------------
// preprocessing kernels (constructor work of pyx:147-209, on the device)
// ------------------------------------------------------------------------------------------------------
__global__ void flags_kernel(const float* __restrict__ data, long long nnz, int* flags) {
  int f = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x) {
    float v = data[i];
    if (v != 1.0f) f |= 1;
    if (v < 0.f) f |= 2;
  }
  f = __reduce_or_sync(0xffffffffu, f);
  if ((threadIdx.x & 31) == 0 && f) atomicOr(flags, f);
}

__global__ void fill_ones_kernel(float* data, long long nnz) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    data[i] = 1.0f;
}

// adjusted cosine: subtract the mean of the stored entries of each row (pyx:277-312); one warp per row
__global__ void row_center_kernel(const int* __restrict__ ptr, float* data, int n_rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_rows) return;
  const int s = ptr[warp], e = ptr[warp + 1];
  if (e <= s) return;
  double sum = 0.0;
  for (int q = s + lane; q < e; q += 32) sum += (double)data[q];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  const double mean = sum / (double)(e - s);
  for (int q = s + lane; q < e; q += 32) data[q] = (float)((double)data[q] - mean);
}

__global__ void col_accum_kernel(const int* __restrict__ idx, const float* __restrict__ data, long long nnz,
                                 double* colsum, double* colsq, int* colcnt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x) {
    const int j = idx[i];
    const double v = (double)data[i];
    if (colsum) atomicAdd(colsum + j, v);
    if (colsq) atomicAdd(colsq + j, v * v);
    if (colcnt) atomicAdd(colcnt + j, 1);
  }
}

// pearson: subtract the per-column mean of stored entries (pyx:236-273)
__global__ void col_center_kernel(const int* __restrict__ idx, float* data, long long nnz,
                                  const double* __restrict__ colsum, const int* __restrict__ colcnt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x) {
    const int j = idx[i];
    const int c = colcnt[j];
    if (c > 0) data[i] = (float)((double)data[i] - colsum[j] / (double)c);
  }
}

// per ORIGINAL column: A (target-side term) and B (neighbour-side term) of the similarity formula
__global__ void norms_kernel(const double* __restrict__ colsq, int n_cols, int mode, float alpha, float* A, float* B,
                             unsigned* Bkey, int* iota) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_cols) return;
  const double sq = colsq[j];
  float a, b;
  if (mode == 0) {  // set kinds: plain sum of squares (pyx:170-174)
    a = b = (float)sq;
  } else if (mode == 1) {  // cosine family
    a = b = (float)sqrt(sq);
  } else {  // asymmetric (pyx:176-180)
    const double n = sqrt(sq) + 1e-6;
    a = (float)pow(n, 2.0 * (double)alpha);
    b = (float)pow(n, 2.0 * (1.0 - (double)alpha));
  }
  A[j] = a;
  B[j] = b;
  Bkey[j] = __float_as_uint(b);  // b >= 0: the bit pattern orders like the value
  iota[j] = j;
}

__global__ void scaled_keys_kernel(const float* __restrict__ B, int n_cols, unsigned* Bkey, int* iota) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_cols) return;
  Bkey[j] = __float_as_uint(fmaxf(B[j], 0.f));
  iota[j] = j;
}

// new numbering: new2old = columns sorted by (B asc, original index asc)
__global__ void renumber_kernel(const int* __restrict__ new2old, const float* __restrict__ A_old,
                                const float* __restrict__ B_old, const int* __restrict__ cnt_old, int n_cols,
                                int* old2new, float* A_new, int2* BN, int* cnt_new) {
  const int jn = blockIdx.x * blockDim.x + threadIdx.x;
  if (jn >= n_cols) return;
  const int jo = new2old[jn];
  old2new[jo] = jn;
  A_new[jn] = A_old[jo];
  BN[jn] = make_int2(__float_as_int(B_old[jo]), jo);
  cnt_new[jn] = cnt_old[jo];
}

__global__ void relabel_kernel(const int* __restrict__ idx_old, const int* __restrict__ old2new, long long nnz, int* idx_new) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    idx_new[i] = old2new[idx_old[i]];
}

__global__ void rowid_iota_kernel(const int* __restrict__ ptr, int n_rows, int* rowid, int* iota) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_rows) return;
  const int s = ptr[warp], e = ptr[warp + 1];
  for (int q = s + lane; q < e; q += 32) { rowid[q] = warp; iota[q] = q; }
}

__global__ void build_csr_ent_kernel(const int* __restrict__ idx, const float* __restrict__ data, long long nnz, int2* ent) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nnz; i += (long long)gridDim.x * blockDim.x)
    ent[i] = make_int2(idx[i], __float_as_int(data[i]));
}

// CSC side: entry q of the column-sorted permutation -> (user, x_ui * w_u)
__global__ void build_csc_kernel(const int* __restrict__ perm, const int* __restrict__ rowid,
                                 const float* __restrict__ data, const float* __restrict__ row_w, long long nnz,
                                 int2* ent, int* idx_only) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x) {
    const int pp = perm[q];
    const int u = rowid[pp];
    if (idx_only) {
      idx_only[q] = u;
    } else {
      float x = data ? data[pp] : 1.0f;
      if (row_w) x *= row_w[u];
      ent[q] = make_int2(u, __float_as_int(x));
    }
  }
}

// split[u*(n_win+1)+w] = first position of row u whose column index >= w*win  (rows are sorted)
__global__ void split_kernel(const int* __restrict__ ptr, const int* __restrict__ idx, int n_rows, int n_win,
                             int win, int* split) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long total = (long long)n_rows * (n_win + 1);
  if (g >= total) return;
  const int u = (int)(g / (n_win + 1)), w = (int)(g % (n_win + 1));
  int lo = ptr[u], hi = ptr[u + 1];
  if (w == 0) { split[g] = lo; return; }
  if (w == n_win) { split[g] = hi; return; }
  const int bound = w * win;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (idx[mid] < bound) lo = mid + 1; else hi = mid;
  }
  split[g] = lo;
}

// Binary path: every (row, window) segment is re-laid 16-byte aligned and padded to a multiple of 4 indices with the
// dummy cell index (w + 1) * win -- one cell past window w's accumulators -- so the accumulate loop has no partial chunks.
__global__ void seg_len_kernel(const int* __restrict__ split, long long n_seg, int n_win, int* len4) {
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= n_seg) return;
  const long long u = g / n_win;
  const int w = (int)(g % n_win);
  const int* sp = split + u * (n_win + 1) + w;
  len4[g] = (sp[1] - sp[0] + 3) & ~3;
}

__global__ void seg_pad_kernel(const int* __restrict__ split, const int* __restrict__ idx, const int* __restrict__ poff,
                               long long n_seg, int n_win, int win, int total, int* idx_pad, int* split_pad) {
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 3;  // 8 lanes per segment
  const int l = threadIdx.x & 7;
  if (g >= n_seg) return;
  const long long u = g / n_win;
  const int w = (int)(g % n_win);
  const int* sp = split + u * (n_win + 1) + w;
  const int s = sp[0], n = sp[1] - sp[0], n4 = (n + 3) & ~3, o = poff[g];
  for (int t = l; t < n4; t += 8) idx_pad[o + t] = t < n ? idx[s + t] : (w + 1) * win;
  if (l == 0) {
    split_pad[u * (n_win + 1) + w] = o;
    if (w == n_win - 1) split_pad[u * (n_win + 1) + n_win] = o + n4;
  }
}

// work[c] = sum over users u of (new) column c of len_u  (the gathered-entry count of SURVEY 8(d))
__global__ void col_work_kernel(const int* __restrict__ csc_ptr, const int* __restrict__ csc_idx,
                                const int2* __restrict__ csc_ent, const int* __restrict__ csr_ptr, int n_cols,
                                unsigned long long* work) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_cols) return;
  unsigned long long s = 0;
  for (int q = csc_ptr[warp] + lane; q < csc_ptr[warp + 1]; q += 32) {
    const int u = csc_idx ? csc_idx[q] : csc_ent[q].x;
    s += (unsigned long long)(csr_ptr[u + 1] - csr_ptr[u]);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) work[warp] = s;
}

}  // namespace sim
}  // namespace b200

using namespace b200;
using namespace b200::sim;

struct b200_sim_s {
  // the launch parameters that do not change from call to call: geometry, formula constants and the handle's buffers
  KParams base{};
  int n_rows = 0;
  long long nnz = 0;
  int kind = 0, normalize = 0;
  float asym_alpha = 0.5f;
  int formula = F_PROD;
  bool binary = false;
  bool pack = false;               // binary path with 16-bit counters (two cells per accumulator word)
  bool allow_pack = true;
  bool scaled = false;             // P3alpha / RP3beta product: CSC values are 1, A and B come from the caller
  const float* h_A = nullptr;
  const float* h_B = nullptr;
  sim_kernel_t kernel = nullptr;   // the window kernel of the formula and counter type
  size_t smem_bytes = 0;
  int n_sm = 0;
  DevBuf<int> csr_ptr, csr_idx, csc_ptr, csc_idx, split, old2new;
  DevBuf<int2> csr_ent, csc_ent, BN;
  DevBuf<float> A, tileB;
  K1DState k1d;                    // binary path, large sparse catalogues (sim_k1d.cuh)
  std::vector<unsigned long long> h_work;  // by ORIGINAL column index
  DevBuf<int> counter, order;
  std::vector<int> h_order;  // cached LPT order for [order_lo, order_hi)
  int order_lo = -1, order_hi = -1;
  bool order_k1c = false;
  DevBuf<unsigned long long> prof;
  bool prof_on = false;
  EpochTimer timer;
};

namespace {

constexpr int GRID1D = 132 * 8;  // grid-stride loops: 8 CTAs per SM of an H100

int bits_for(long long n) {
  int b = 1;
  while ((1ll << b) < n) ++b;
  return b;
}

void build(b200_sim_s* h, const int32_t* h_indptr, const int32_t* h_indices, const float* h_data,
           const float* h_row_weights, cudaStream_t st) {
  KParams& b = h->base;
  const int n_rows = h->n_rows, n_cols = b.n_cols;
  const long long nnz = h->nnz;
  const size_t nnz1 = (size_t)std::max<long long>(nnz, 1);
  h->n_sm = sm_count();

  h->csr_ptr.alloc((size_t)n_rows + 1);
  DevBuf<int> idx_old(nnz1);
  DevBuf<float> data(nnz1);
  B200_CUDA(cudaMemcpyAsync(h->csr_ptr.get(), h_indptr, sizeof(int) * ((size_t)n_rows + 1), cudaMemcpyHostToDevice, st));
  if (nnz) {
    B200_CUDA(cudaMemcpyAsync(idx_old.get(), h_indices, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(data.get(), h_data, sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, st));
  }
  DevBuf<float> row_w;
  if (h_row_weights) {
    row_w.alloc((size_t)n_rows);
    B200_CUDA(cudaMemcpyAsync(row_w.get(), h_row_weights, sizeof(float) * (size_t)n_rows, cudaMemcpyHostToDevice, st));
  }

  // ---- per-kind data transform (pyx:160-165)
  const bool set_kind = !h->scaled && (h->kind == B200_SIM_JACCARD || h->kind == B200_SIM_DICE || h->kind == B200_SIM_TVERSKY);
  DevBuf<double> colsum((size_t)n_cols), colsq((size_t)n_cols);
  DevBuf<int> colcnt((size_t)n_cols);
  B200_CUDA(cudaMemsetAsync(colsum.get(), 0, sizeof(double) * (size_t)n_cols, st));
  B200_CUDA(cudaMemsetAsync(colsq.get(), 0, sizeof(double) * (size_t)n_cols, st));
  B200_CUDA(cudaMemsetAsync(colcnt.get(), 0, sizeof(int) * (size_t)n_cols, st));
  if (nnz && !h->scaled) {
    if (set_kind) {
      fill_ones_kernel<<<GRID1D, 256, 0, st>>>(data.get(), nnz); count_launch();
    } else if (h->kind == B200_SIM_ADJUSTED) {
      row_center_kernel<<<div_up((long long)n_rows * 32, 256), 256, 0, st>>>(h->csr_ptr.get(), data.get(), n_rows); count_launch();
    } else if (h->kind == B200_SIM_PEARSON) {
      col_accum_kernel<<<GRID1D, 256, 0, st>>>(idx_old.get(), data.get(), nnz, colsum.get(), nullptr, colcnt.get()); count_launch();
      col_center_kernel<<<GRID1D, 256, 0, st>>>(idx_old.get(), data.get(), nnz, colsum.get(), colcnt.get()); count_launch();
      B200_CUDA(cudaMemsetAsync(colcnt.get(), 0, sizeof(int) * (size_t)n_cols, st));
    }
  }
  // ---- flags: binary path (every stored value == 1, no row weights), signed data
  DevBuf<int> flags(1);
  B200_CUDA(cudaMemsetAsync(flags.get(), 0, sizeof(int), st));
  if (nnz) { flags_kernel<<<GRID1D, 256, 0, st>>>(data.get(), nnz, flags.get()); count_launch(); }
  int hflags = 0;
  B200_CUDA(cudaMemcpyAsync(&hflags, flags.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  // ---- column sums of squares (before the row weights, pyx:169-194), counts, formula terms
  if (nnz) { col_accum_kernel<<<GRID1D, 256, 0, st>>>(idx_old.get(), data.get(), nnz, nullptr, colsq.get(), colcnt.get()); count_launch(); }
  DevBuf<float> A_old((size_t)n_cols), B_old((size_t)n_cols);
  DevBuf<unsigned> Bkey((size_t)n_cols), Bkey_sorted((size_t)n_cols);
  DevBuf<int> col_iota((size_t)n_cols), new2old((size_t)n_cols), cnt_new((size_t)n_cols);
  if (h->scaled) {
    B200_CUDA(cudaMemcpyAsync(A_old.get(), h->h_A, sizeof(float) * (size_t)n_cols, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(B_old.get(), h->h_B, sizeof(float) * (size_t)n_cols, cudaMemcpyHostToDevice, st));
    scaled_keys_kernel<<<div_up(n_cols, 256), 256, 0, st>>>(B_old.get(), n_cols, Bkey.get(), col_iota.get());
  } else {
    // euclidean keeps the plain sums of squares too (Compute_Similarity_Euclidean.py:112)
    const int norm_mode = (set_kind || h->kind == B200_SIM_EUCLIDEAN) ? 0 : (h->kind == B200_SIM_ASYMMETRIC ? 2 : 1);
    norms_kernel<<<div_up(n_cols, 256), 256, 0, st>>>(colsq.get(), n_cols, norm_mode, h->asym_alpha, A_old.get(), B_old.get(),
                                                      Bkey.get(), col_iota.get());
  }
  count_launch();

  // ---- renumber the columns by (B asc, original index asc): stable radix sort on the float bit pattern
  {
    size_t tb = 0;
    B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, Bkey.get(), Bkey_sorted.get(), col_iota.get(), new2old.get(), n_cols, 0, 32, st));
    DevBuf<unsigned char> tmp(tb + 16);
    B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tb, Bkey.get(), Bkey_sorted.get(), col_iota.get(), new2old.get(), n_cols, 0, 32, st));
    count_launch(4);
    B200_CUDA(cudaStreamSynchronize(st));
  }
  h->old2new.alloc((size_t)n_cols);
  h->A.alloc((size_t)n_cols);
  h->BN.alloc((size_t)n_cols);
  renumber_kernel<<<div_up(n_cols, 256), 256, 0, st>>>(new2old.get(), A_old.get(), B_old.get(), colcnt.get(), n_cols,
                                                       h->old2new.get(), h->A.get(), h->BN.get(), cnt_new.get());
  count_launch();
  B200_CUDA(cudaStreamSynchronize(st));
  b.eu_signed = (hflags & 2) != 0;
  h->binary = ((hflags & 1) == 0) && !h_row_weights && !h->scaled;

  // ---- CSR in the new numbering: relabel, then sort every row segment by the new index
  h->csr_idx.alloc(nnz1 + 8);
  DevBuf<float> data_sorted(nnz1);
  if (nnz) {
    DevBuf<int> idx_new(nnz1);
    relabel_kernel<<<GRID1D, 256, 0, st>>>(idx_old.get(), h->old2new.get(), nnz, idx_new.get()); count_launch();
    size_t tb = 0;
    B200_CUDA(cub::DeviceSegmentedSort::SortPairs(nullptr, tb, idx_new.get(), h->csr_idx.get(), data.get(), data_sorted.get(),
                                                  (long long)nnz, (long long)n_rows, h->csr_ptr.get(), h->csr_ptr.get() + 1, st));
    DevBuf<unsigned char> tmp(tb + 16);
    B200_CUDA(cub::DeviceSegmentedSort::SortPairs(tmp.get(), tb, idx_new.get(), h->csr_idx.get(), data.get(), data_sorted.get(),
                                                  (long long)nnz, (long long)n_rows, h->csr_ptr.get(), h->csr_ptr.get() + 1, st));
    count_launch(3);
    B200_CUDA(cudaStreamSynchronize(st));
  }
  idx_old.release();
  data.release();

  // ---- CSC (new numbering): exclusive scan of the column counts, stable sort of (column, position) pairs
  h->csc_ptr.alloc((size_t)n_cols + 1);
  B200_CUDA(cudaMemsetAsync(h->csc_ptr.get(), 0, sizeof(int) * ((size_t)n_cols + 1), st));
  {
    size_t tb = 0;
    B200_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, cnt_new.get(), h->csc_ptr.get() + 1, n_cols, st));
    DevBuf<unsigned char> tmp(tb + 16);
    B200_CUDA(cub::DeviceScan::InclusiveSum(tmp.get(), tb, cnt_new.get(), h->csc_ptr.get() + 1, n_cols, st));
    count_launch(2);
    B200_CUDA(cudaStreamSynchronize(st));
  }
  DevBuf<int> csc_pos;  // binary path: CSR position of every CSC entry (its place in the user's sorted row), for K1-D
  if (nnz) {
    DevBuf<int> rowid(nnz1), iota(nnz1), keys_out(nnz1), perm(nnz1);
    rowid_iota_kernel<<<div_up((long long)n_rows * 32, 256), 256, 0, st>>>(h->csr_ptr.get(), n_rows, rowid.get(), iota.get()); count_launch();
    size_t tb = 0;
    const int end_bit = bits_for(n_cols);
    B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, h->csr_idx.get(), keys_out.get(), iota.get(), perm.get(), (int)nnz, 0, end_bit, st));
    DevBuf<unsigned char> tmp(tb + 16);
    B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tb, h->csr_idx.get(), keys_out.get(), iota.get(), perm.get(), (int)nnz, 0, end_bit, st));
    count_launch(4);
    if (h->binary) {
      h->csc_idx.alloc((size_t)nnz);
      build_csc_kernel<<<GRID1D, 256, 0, st>>>(perm.get(), rowid.get(), data_sorted.get(), nullptr, nnz, nullptr, h->csc_idx.get());
      csc_pos = std::move(perm);
    } else {
      h->csc_ent.alloc((size_t)nnz);
      h->csr_ent.alloc((size_t)nnz + 8);
      build_csc_kernel<<<GRID1D, 256, 0, st>>>(perm.get(), rowid.get(), h->scaled ? nullptr : data_sorted.get(), row_w.get(), nnz, h->csc_ent.get(), nullptr);
      build_csr_ent_kernel<<<GRID1D, 256, 0, st>>>(h->csr_idx.get(), data_sorted.get(), nnz, h->csr_ent.get()); count_launch();
    }
    count_launch();
    B200_CUDA(cudaStreamSynchronize(st));
  }

  if (h->scaled) {
    h->formula = F_SCALE;
  } else if (set_kind) {
    h->formula = h->kind == B200_SIM_JACCARD ? F_JACCARD : (h->kind == B200_SIM_DICE ? F_DICE : F_TVERSKY);
  } else if (h->kind == B200_SIM_EUCLIDEAN) {
    h->formula = F_EUCLID;
  } else {
    h->formula = h->normalize ? F_PROD : F_NONORM;
  }
  b.signed_data = (b.eu_signed && h->formula != F_EUCLID) ? 1 : 0;  // euclidean similarities are never negative

  // ---- window geometry: the accumulator covers `win` neighbour columns; n_win passes per target column
  int dev = 0, max_smem = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  int cap = 2048;
  while (cap < 4 * b.K) cap <<= 1;
  B200_REQUIRE(cap <= 8192, "topK=%d too large for the top-K kernel (max 2048); use the dense path", b.K);
  b.cap = cap;
  b.cap_alloc = cap;
  const size_t staging = (size_t)STAGE_INTS * 4;
  // binary path: counts fit 15 bits when no column holds 32768 entries (a dot product is at most the shorter column)
  {
    std::vector<int> hcnt((size_t)n_cols);
    B200_CUDA(cudaMemcpy(hcnt.data(), cnt_new.get(), sizeof(int) * (size_t)n_cols, cudaMemcpyDeviceToHost));
    int mx = 0;
    for (int j = 0; j < n_cols; ++j) mx = std::max(mx, hcnt[(size_t)j]);
    h->pack = h->binary && mx < 32768 && h->allow_pack;  // half_ge_mask needs counts below 0x8000
  }
  auto windows_needed = [&](int cells_per_word, long long* cells_out) {
    int nw = 1;
    long long mc = 0;
    for (;; ++nw) {  // the tile-bound table grows with the window count
      const size_t fixed = (size_t)cap * 8 + staging + (size_t)nw * (MAXTILES + 1) * 4 + sizeof(Shared) + 1024;
      mc = (((long long)max_smem - (long long)fixed) / 4) * cells_per_word;
      mc = std::min<long long>(mc, (long long)MAXTILES * THREADS * 4 * cells_per_word);
      B200_REQUIRE(mc >= 4096, "not enough shared memory (%d bytes) for the similarity kernel", max_smem);
      if ((long long)nw * mc >= n_cols) break;
    }
    *cells_out = mc;
    return nw;
  };
  long long max_cells = 0, max_cells_unpacked = 0;
  const int n_win_unpacked = windows_needed(1, &max_cells_unpacked);
  if (h->pack && windows_needed(2, &max_cells) >= n_win_unpacked) h->pack = false;  // 16-bit counters only pay off with fewer windows
  const int cpw = h->pack ? 2 : 1;       // cells per 4-byte accumulator word
  const int cpv = 4 * cpw;               // cells per 16-byte vector
  const int tile = THREADS * cpv;        // cells per block-wide scan iteration
  int n_win = windows_needed(cpw, &max_cells);
  int win = (n_cols + n_win - 1) / n_win;
  win = (win + cpv - 1) / cpv * cpv;
  if (win < cpv) win = cpv;
  b.n_win = n_win;
  b.win = win;
  b.acc_cells = std::max(win / cpw, SBINS) + 4;  // + the dummy cell the padded row segments point at (cell index `win`)
  h->smem_bytes = (size_t)b.acc_cells * 4 + (size_t)cap * 8 + staging + (size_t)n_win * (MAXTILES + 1) * 4;
  const bool binary = h->binary, pack = h->pack;
  h->kernel = with_formula<F_PROD, F_NONORM, F_JACCARD, F_DICE, F_SCALE, F_EUCLID, F_TVERSKY>(h->formula, [&](auto f) -> sim_kernel_t {
    constexpr int F = decltype(f)::value;
    if constexpr (F == F_SCALE) return sim_topk_kernel<F, false, false>;  // never binary: A and B are the caller's
    else return binary ? (pack ? sim_topk_kernel<F, true, true> : sim_topk_kernel<F, true, false>) : sim_topk_kernel<F, false, false>;
  });
  raise_smem_limit(h->kernel, h->smem_bytes);
  h->tileB.alloc((size_t)n_win * (MAXTILES + 1));
  tile_bounds_kernel<<<div_up((long long)n_win * (MAXTILES + 1), 128), 128, 0, st>>>(h->BN.get(), n_cols, n_win, win, tile, h->tileB.get());
  count_launch();
  {
    // lanes per row segment in the accumulate phase: enough 16-byte chunks for the average segment
    const double avg_seg = nnz > 0 ? (double)nnz / (double)n_rows / (double)n_win : 1.0;
    const double chunks = avg_seg / (h->binary ? 4.0 : 2.0) + 1.0;
    int l2 = 1;
    while (l2 < 5 && (1 << l2) < chunks) ++l2;
    b.lpu_log2 = l2;
  }
  if (n_win > 1 || h->binary) {
    h->split.alloc((size_t)n_rows * (n_win + 1));
    const long long total = (long long)n_rows * (n_win + 1);
    split_kernel<<<div_up(total, 256), 256, 0, st>>>(h->csr_ptr.get(), h->csr_idx.get(), n_rows, n_win, win, h->split.get()); count_launch();
  }
  DevBuf<int> idx_pad, split_pad;
  if (h->binary) {  // padded, 16-byte aligned (row, window) segments
    const long long n_seg = (long long)n_rows * n_win;
    B200_REQUIRE((long long)nnz + 3 * n_seg < (1ll << 31), "matrix too large for 32-bit positions in the padded row layout");
    DevBuf<int> len4((size_t)n_seg + 1), poff((size_t)n_seg + 1);
    B200_CUDA(cudaMemsetAsync(len4.get() + n_seg, 0, sizeof(int), st));
    seg_len_kernel<<<div_up(n_seg, 256), 256, 0, st>>>(h->split.get(), n_seg, n_win, len4.get()); count_launch();
    size_t tb = 0;
    B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, len4.get(), poff.get(), (int)(n_seg + 1), st));
    DevBuf<unsigned char> tmp(tb);
    B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, len4.get(), poff.get(), (int)(n_seg + 1), st)); count_launch();
    int total_pad = 0;
    B200_CUDA(cudaMemcpyAsync(&total_pad, poff.get() + n_seg, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    idx_pad.alloc((size_t)total_pad + 8);
    split_pad.alloc((size_t)n_rows * (n_win + 1));
    seg_pad_kernel<<<div_up(n_seg * 8, 256), 256, 0, st>>>(h->split.get(), h->csr_idx.get(), poff.get(), n_seg, n_win, win, total_pad,
                                                          idx_pad.get(), split_pad.get()); count_launch();
    B200_CUDA(cudaStreamSynchronize(st));
  }
  // ---- per-column work (for LPT ordering and the bytes model), reported by ORIGINAL column index
  {
    DevBuf<unsigned long long> work((size_t)n_cols);
    col_work_kernel<<<div_up((long long)n_cols * 32, 256), 256, 0, st>>>(h->csc_ptr.get(), h->binary ? h->csc_idx.get() : nullptr,
                                                                        h->binary ? nullptr : h->csc_ent.get(), h->csr_ptr.get(), n_cols, work.get());
    count_launch();
    std::vector<unsigned long long> w_new((size_t)n_cols);
    std::vector<int> o2n((size_t)n_cols);
    B200_CUDA(cudaMemcpyAsync(w_new.data(), work.get(), sizeof(unsigned long long) * (size_t)n_cols, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(o2n.data(), h->old2new.get(), sizeof(int) * (size_t)n_cols, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    h->h_work.resize((size_t)n_cols);
    for (int c = 0; c < n_cols; ++c) h->h_work[(size_t)c] = w_new[(size_t)o2n[(size_t)c]];
  }
  k1d_build(h, cnt_new.get(), csc_pos.get(), st);
  csc_pos.release();
  if (h->binary) {
    h->csr_idx = std::move(idx_pad);
    h->split = std::move(split_pad);
  } else {
    h->csr_idx.release();  // the AoS copy carries the indices
  }
  h->counter.alloc(1);
  h->order.alloc((size_t)n_cols);
  b.csr_ptr = h->csr_ptr.get(); b.csr_ent = h->csr_ent.get(); b.csr_idx = h->csr_idx.get();
  b.split = h->split.get();
  b.csc_ptr = h->csc_ptr.get(); b.csc_ent = h->csc_ent.get(); b.csc_idx = h->csc_idx.get();
  b.A = h->A.get(); b.BN = h->BN.get(); b.tileB = h->tileB.get(); b.old2new = h->old2new.get();
  b.order = h->order.get(); b.redo = h->order.get(); b.counter = h->counter.get();
}

}  // namespace

namespace {

// The steps every create entry point shares: the checks of the shape and the input arrays, the environment hooks, a new
// handle that `init` fills with the fields of its kind (and may reject), build(); the handle is deleted when a step fails.
template <class Init>
int create(const char* fn, b200_sim_t* out, int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* h_indptr,
           const int32_t* h_indices, const float* h_data, int topK, float shrink, const float* h_row_weights, void* stream,
           Init init) {
  if (out) *out = nullptr;
  b200_sim_s* h = nullptr;
  int rc = guarded([&] {
    B200_REQUIRE(out != nullptr, "%s: out is NULL", fn);
    B200_REQUIRE(n_rows > 0 && n_cols > 0 && nnz >= 0, "%s: bad shape %lld x %lld nnz %lld", fn, (long long)n_rows,
                 (long long)n_cols, (long long)nnz);
    B200_REQUIRE(n_rows < (1ll << 31) - 1 && n_cols < (1ll << 31) - 1 && nnz < (1ll << 31) - 1, "%s: int32 index range exceeded", fn);
    B200_REQUIRE(topK >= 1, "%s: topK must be >= 1", fn);
    B200_REQUIRE(h_indptr && (nnz == 0 || (h_indices && h_data)), "%s: NULL input array", fn);
    h = new b200_sim_s();
    h->allow_pack = getenv("B200REC_NO_PACK") == nullptr;  // test hook: force 32-bit counters on the binary path
    // K1-D routing: on by default for binary data with >= k1c_min_cols columns; B200REC_K1C=0 disables it, the other two
    // variables are test hooks (small matrices, forced overflow -> redo path)
    if (const char* e = getenv("B200REC_K1C")) h->k1d.want_k1c = atoi(e) != 0;
    if (const char* e = getenv("B200REC_K1C_LAMBDA")) h->k1d.k1c_lambda = atof(e);
    if (const char* e = getenv("B200REC_K1C_MINCOLS")) h->k1d.k1c_min_cols = atoi(e);
    h->n_rows = (int)n_rows;
    h->nnz = nnz;
    KParams& b = h->base;
    b.n_cols = (int)n_cols;
    b.K = (int)std::min<int64_t>(topK, n_cols);
    b.se = shrink + 1e-6f;
    b.shrink_div = shrink != 0.f ? shrink : 1.f;
    b.eu_shrink = shrink;
    b.ta = b.tb = 1.f;
    b.eu_mode = B200_EUCLID_LIN;
    b.eu_div = 1.f;
    init(h);
    build(h, h_indptr, h_indices, h_data, h_row_weights, (cudaStream_t)stream);
    h->h_A = h->h_B = nullptr;  // the caller's arrays, read by build() only
    *out = h;
  });
  if (rc != B200_OK) delete h;
  return rc;
}

void check_range(const b200_sim_s* h, int start_col, int end_col, const char* fn) {
  B200_REQUIRE(0 <= start_col && start_col <= end_col && end_col <= h->base.n_cols, "%s: bad column range [%d,%d)", fn,
               start_col, end_col);
}

}  // namespace

extern "C" {

int b200_sim_create(b200_sim_t* out, int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* h_indptr,
                    const int32_t* h_indices, const float* h_data, int kind, int topK, float shrink, int normalize,
                    float asymmetric_alpha, float tversky_alpha, float tversky_beta, const float* h_row_weights,
                    void* stream) {
  return create("b200_sim_create", out, n_rows, n_cols, nnz, h_indptr, h_indices, h_data, topK, shrink, h_row_weights, stream,
                [&](b200_sim_s* h) {
    B200_REQUIRE(kind >= B200_SIM_COSINE && kind <= B200_SIM_TVERSKY, "b200_sim_create: unknown similarity kind %d", kind);
    h->kind = kind;
    const bool set_kind = kind == B200_SIM_JACCARD || kind == B200_SIM_DICE || kind == B200_SIM_TVERSKY;
    h->normalize = set_kind ? 0 : (normalize != 0);
    h->asym_alpha = asymmetric_alpha;
    h->base.ta = tversky_alpha;
    h->base.tb = tversky_beta;
  });
}

int b200_sim_create_scaled(b200_sim_t* out, int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* h_indptr,
                           const int32_t* h_indices, const float* h_data, const float* h_A, const float* h_B, int topK,
                           void* stream) {
  return create("b200_sim_create_scaled", out, n_rows, n_cols, nnz, h_indptr, h_indices, h_data, topK, 0.f, nullptr, stream,
                [&](b200_sim_s* h) {
    B200_REQUIRE(h_A && h_B, "b200_sim_create_scaled: NULL argument");
    h->kind = B200_SIM_COSINE;
    h->scaled = true;
    h->h_A = h_A; h->h_B = h_B;
  });
}

int b200_sim_create_euclidean(b200_sim_t* out, int64_t n_rows, int64_t n_cols, int64_t nnz, const int32_t* h_indptr,
                              const int32_t* h_indices, const float* h_data, int topK, float shrink, int normalize,
                              int normalize_avg_row, int distance_mode, void* stream) {
  return create("b200_sim_create_euclidean", out, n_rows, n_cols, nnz, h_indptr, h_indices, h_data, topK, shrink, nullptr, stream,
                [&](b200_sim_s* h) {
    B200_REQUIRE(distance_mode >= B200_EUCLID_EXP && distance_mode <= B200_EUCLID_LOG,
                 "b200_sim_create_euclidean: unknown similarity_from_distance_mode %d", distance_mode);
    h->kind = B200_SIM_EUCLIDEAN;
    h->base.eu_mode = distance_mode;
    h->base.eu_norm = normalize != 0;
    h->base.eu_div = normalize_avg_row ? (float)h->n_rows : 1.f;
  });
}

int b200_sim_destroy(b200_sim_t h) {
  if (!h) return B200_OK;
  delete h;
  return B200_OK;
}

int b200_sim_info(b200_sim_t h, int* K, int* n_windows, int* window_cells, int* binary_path, int* signed_data) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_info: NULL handle");
    if (K) *K = h->base.K;
    if (n_windows) *n_windows = h->base.n_win;
    if (window_cells) *window_cells = h->base.win;
    if (binary_path) *binary_path = h->binary ? (h->pack ? 2 : 1) : 0;
    if (signed_data) *signed_data = h->base.eu_signed;
  });
}

struct PeerOut { int* idx; float* val; int* cnt; };

static void launch_topk(b200_sim_t h, int start_col, int end_col, int32_t* d_idx, float* d_val, int32_t* d_cnt, float* d_dense,
                        cudaStream_t st, const PeerOut* peers = nullptr, int n_peers = 0) {
  K1DState& k = h->k1d;
  const int n_cols = h->base.n_cols, n_range = end_col - start_col;
  const bool use_k1c = k.k1c && d_dense == nullptr;
  // Routing + longest-processing-time-first order of the local columns (cached per range).  With K1-D the columns whose
  // expected hits per neighbour (gathered entries / n_cols) stay below k1c_lambda go to the nibble-counter kernel (`worklist`);
  // the rest -- and whatever that kernel hands back -- go to the window kernel (`order`).
  if (h->order_lo != start_col || h->order_hi != end_col || h->order_k1c != use_k1c) {
    const unsigned long long* w = h->h_work.data() + start_col;
    std::vector<int> sparse;
    h->h_order.clear();
    int n_nonempty_dense = 0;
    for (int i = 0; i < n_range; ++i) {
      const bool sp = use_k1c && w[i] > 0 && (double)w[i] <= k.k1c_lambda * (double)n_cols;
      (sp ? sparse : h->h_order).push_back(i);
      if (!sp && w[i] > 0) ++n_nonempty_dense;
    }
    // the pair path needs every pair's pass in this call: the whole column range, every non-empty column on K1-D
    k.pair_path_last = k.ctas_up > 0 && use_k1c && start_col == 0 && end_col == n_cols && n_nonempty_dense == 0 && !sparse.empty();
    auto by_work = [w](int a, int b) { return w[a] > w[b]; };
    std::stable_sort(h->h_order.begin(), h->h_order.end(), by_work);
    std::stable_sort(sparse.begin(), sparse.end(), by_work);
    k.n_dense_last = (int)h->h_order.size();
    k.n_sparse_last = (int)sparse.size();
    if (!h->h_order.empty())
      B200_CUDA(cudaMemcpyAsync(h->order.get(), h->h_order.data(), sizeof(int) * h->h_order.size(), cudaMemcpyHostToDevice, st));
    std::vector<int4> wl(sparse.size());
    for (size_t i = 0; i < sparse.size(); ++i) {
      const int cn = k.h_old2new[(size_t)(start_col + sparse[i])];
      wl[i] = make_int4(cn, sparse[i], k.h_csc_ptr[(size_t)cn], k.h_csc_ptr[(size_t)cn + 1]);
    }
    if (!wl.empty()) B200_CUDA(cudaMemcpyAsync(k.worklist.get(), wl.data(), sizeof(int4) * wl.size(), cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));
    h->order_lo = start_col;
    h->order_hi = end_col;
    h->order_k1c = use_k1c;
  }
  const bool pair_path = k.pair_path_last && n_peers == 0;
  const int n_sparse = use_k1c ? k.n_sparse_last : 0, n_dense = use_k1c ? k.n_dense_last : n_range;
  B200_CUDA(cudaMemsetAsync(h->counter.get(), 0, sizeof(int), st));
  if (pair_path) k1d_pair_buffers(h, st);
  KParams p = h->base;
  p.col_begin = start_col; p.n_range = n_dense;
  p.n_out = 1 + n_peers;
  p.o_idx[0] = d_idx; p.o_val[0] = d_val; p.o_cnt[0] = d_cnt;
  for (int r = 0; r < n_peers; ++r) { p.o_idx[1 + r] = peers[r].idx; p.o_val[1 + r] = peers[r].val; p.o_cnt[1 + r] = peers[r].cnt; }
  p.dense_out = d_dense;
  p.prof = h->prof_on ? h->prof.get() : nullptr;
  p.n_range_dev = nullptr;
  h->timer.begin(st);
  if (n_sparse > 0) k1d_launch(h, p, n_sparse, pair_path, st);  // the pair path implies n_sparse > 0
  if (n_dense > 0 || n_sparse > 0) {
    const int grid = n_sparse > 0 ? h->n_sm : std::min(n_dense, h->n_sm);
    h->kernel<<<grid, THREADS, h->smem_bytes, st>>>(p);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  h->timer.end(st);
}

int b200_sim_compute_device(b200_sim_t h, int start_col, int end_col, int32_t* d_idx, float* d_val, int32_t* d_cnt,
                            void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_compute: NULL handle");
    check_range(h, start_col, end_col, "b200_sim_compute");
    if (end_col == start_col) return;
    B200_REQUIRE(d_idx && d_val && d_cnt, "b200_sim_compute: NULL output");
    launch_topk(h, start_col, end_col, d_idx, d_val, d_cnt, nullptr, (cudaStream_t)stream);
  });
}

int b200_sim_compute_peers_device(b200_sim_t h, int start_col, int end_col, int n_tables, void* const* d_tables, int64_t idx_offset,
                                  int64_t val_offset, int64_t cnt_offset, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_compute_peers: NULL handle");
    check_range(h, start_col, end_col, "b200_sim_compute_peers");
    B200_REQUIRE(n_tables >= 1 && n_tables <= B200_MAX_PEERS && d_tables != nullptr, "b200_sim_compute_peers: 1..%d tables", B200_MAX_PEERS);
    if (end_col == start_col) return;
    PeerOut out[B200_MAX_PEERS];
    for (int r = 0; r < n_tables; ++r) {
      B200_REQUIRE(d_tables[r] != nullptr, "b200_sim_compute_peers: NULL table");
      int32_t* base = reinterpret_cast<int32_t*>(d_tables[r]);
      // rows are addressed by GLOBAL column: the range's first row sits at start_col
      out[r].idx = base + idx_offset + (int64_t)start_col * h->base.K;
      out[r].val = reinterpret_cast<float*>(base + val_offset) + (int64_t)start_col * h->base.K;
      out[r].cnt = base + cnt_offset + start_col;
    }
    launch_topk(h, start_col, end_col, out[0].idx, out[0].val, out[0].cnt, nullptr, (cudaStream_t)stream, out + 1, n_tables - 1);
  });
}

int b200_sim_compute_dense_device(b200_sim_t h, int start_col, int end_col, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_compute_dense: NULL handle");
    B200_REQUIRE(h->formula != F_EUCLID, "b200_sim_compute_dense: the euclidean similarity has no dense output mode");
    check_range(h, start_col, end_col, "b200_sim_compute_dense");
    if (end_col == start_col) return;  // an empty range has an empty output, which may well be a NULL pointer
    B200_REQUIRE(d_out != nullptr, "b200_sim_compute_dense: NULL output");
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * (size_t)(end_col - start_col) * (size_t)h->base.n_cols, st));
    launch_topk(h, start_col, end_col, nullptr, nullptr, nullptr, d_out, st);
  });
}

int b200_sim_compute(b200_sim_t h, int start_col, int end_col, int32_t* h_idx, float* h_val, int32_t* h_cnt) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_compute: NULL handle");
    check_range(h, start_col, end_col, "b200_sim_compute");
    const size_t n_range = (size_t)(end_col - start_col), K = (size_t)h->base.K;
    if (n_range == 0) return;
    DevBuf<int> d_idx(n_range * K), d_cnt(n_range);
    DevBuf<float> d_val(n_range * K);
    int rc = b200_sim_compute_device(h, start_col, end_col, d_idx.get(), d_val.get(), d_cnt.get(), nullptr);
    if (rc != B200_OK) throw CudaFail{rc};
    B200_CUDA(cudaMemcpy(h_idx, d_idx.get(), sizeof(int) * n_range * K, cudaMemcpyDeviceToHost));
    B200_CUDA(cudaMemcpy(h_val, d_val.get(), sizeof(float) * n_range * K, cudaMemcpyDeviceToHost));
    B200_CUDA(cudaMemcpy(h_cnt, d_cnt.get(), sizeof(int) * n_range, cudaMemcpyDeviceToHost));
  });
}

int b200_sim_debug_set_cap(b200_sim_t h, int cap) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_debug_set_cap: NULL handle");
    B200_REQUIRE(cap > h->base.K && cap <= h->base.cap_alloc, "b200_sim_debug_set_cap: cap must be in (K, %d]", h->base.cap_alloc);
    h->base.cap = cap;
  });
}

int b200_sim_debug_phase_cycles(b200_sim_t h, int enable, uint64_t* out16) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_debug_phase_cycles: NULL handle");
    if (h->prof.n == 0) {
      h->prof.alloc(16);
      B200_CUDA(cudaMemset(h->prof.get(), 0, 16 * sizeof(unsigned long long)));
    }
    if (out16) {
      B200_CUDA(cudaDeviceSynchronize());
      B200_CUDA(cudaMemcpy(out16, h->prof.get(), 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      B200_CUDA(cudaMemset(h->prof.get(), 0, 16 * sizeof(unsigned long long)));
    }
    h->prof_on = enable != 0;
  });
}

int b200_sim_debug_k1c(b200_sim_t h, int set_fail_every, int* enabled, int* ctas_per_sm, int* n_bitmap_cols, int* n_window_cols) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_debug_k1c: NULL handle");
    const K1DState& k = h->k1d;
    if (set_fail_every >= 0 && k.k1c) h->base.fail_every = set_fail_every;  // 0 = off; n: every n-th local column is handed back
    if (enabled) *enabled = k.k1c ? 1 : 0;
    if (ctas_per_sm) *ctas_per_sm = k.k1c ? k.ctas_per_sm : 0;
    if (n_bitmap_cols) *n_bitmap_cols = k.n_sparse_last;  // routing of the last launch
    if (n_window_cols) {
      *n_window_cols = k.n_dense_last;
      if (k.k1c && k.n_sparse_last > 0) {  // the nibble kernel's redo count is on the device
        B200_CUDA(cudaDeviceSynchronize());
        B200_CUDA(cudaMemcpy(n_window_cols, k.fail.get(), sizeof(int), cudaMemcpyDeviceToHost));
      }
    }
  });
}

int b200_sim_debug_pair_lists(b200_sim_t h, int set_tile_log2, int* tile_log2, int32_t* deg, int32_t* mir_off) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_sim_debug_pair_lists: NULL handle");
    K1DState& k = h->k1d;
    if (set_tile_log2 >= 0) {
      B200_REQUIRE(set_tile_log2 <= 12, "b200_sim_debug_pair_lists: tile_log2 must be in [0, 12]");
      k.tile_log2_req = set_tile_log2;
      k.tile_fill.release();  // the next pair-path call sizes the tiles again
      h->base.tile_fill = nullptr;
    }
    if (tile_log2) *tile_log2 = h->base.tile_log2;
    if (deg || mir_off) {
      B200_REQUIRE(k.deg.n > 0, "b200_sim_debug_pair_lists: no call has taken the pair path yet");
      B200_CUDA(cudaDeviceSynchronize());
      const size_t bytes = sizeof(int) * ((size_t)h->base.n_cols + 1);
      if (deg) B200_CUDA(cudaMemcpy(deg, k.deg.get(), bytes, cudaMemcpyDeviceToHost));
      if (mir_off) B200_CUDA(cudaMemcpy(mir_off, k.mir_off.get(), bytes, cudaMemcpyDeviceToHost));
    }
  });
}

int b200_sim_last_kernel_ms(b200_sim_t h, float* ms) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr && ms != nullptr, "b200_sim_last_kernel_ms: NULL argument");
    B200_REQUIRE(h->timer.timed, "b200_sim_last_kernel_ms: no kernel launched yet");
    h->timer.elapsed(ms);
  });
}

int b200_sim_col_work(b200_sim_t h, int64_t* out_n_cols) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr && out_n_cols != nullptr, "b200_sim_col_work: NULL argument");
    for (int c = 0; c < h->base.n_cols; ++c) out_n_cols[c] = (int64_t)h->h_work[(size_t)c];
  });
}

int b200_sim_work(b200_sim_t h, int start_col, int end_col, int64_t* gathered_entries) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr && gathered_entries != nullptr, "b200_sim_work: NULL argument");
    check_range(h, start_col, end_col, "b200_sim_work");
    unsigned long long s = 0;
    for (int c = start_col; c < end_col; ++c) s += h->h_work[(size_t)c];
    *gathered_entries = (int64_t)s;
  });
}

}  // extern "C"
