// The top-K selections' shared parts: the orderable bit map of a float, the keys built from it, and the MSB-first radix
// select that finds the K-th largest key.
//
// A key is an unsigned integer whose order is the order the caller ranks by: the ordered value bits in the high word, a
// tie-break (usually ~index, so that ties go to the ascending index) in the low word.  The select finds the K-th largest
// of n keys one digit at a time from the top: clear a histogram, count the digit of every key that matches the prefix fixed
// so far, find the bin that holds the need-th largest key, fix that digit, repeat.  It stops as soon as the bin is kept
// whole: every key with the prefix survives, and the undecided low digits of the threshold stay zero, so that exactly the
// K largest keys are >= it.
#pragma once

#include "common.cuh"

namespace b200 {

typedef unsigned long long u64;

// Unsigned order = float order: +0 above -0, +NaN above +inf and -NaN below -inf.  Callers that rank NaN or -0 otherwise
// apply their rule before or after this map.
__device__ __forceinline__ unsigned orderable(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ u64 orderable(double v) {
  const u64 b = (u64)__double_as_longlong(v);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// The key of value v at index qi in a line of the top-K selections (dense_topk.cu, the sparse SLIM ElasticNet solve): the
// value bits, then ~index so that ties go to the ascending index.  orderable() maps +NaN above +inf and -NaN below -inf;
// every NaN is moved to one end instead, by mode.
__device__ __forceinline__ u64 line_key(float v, int qi, bool nan_high) {
  const unsigned o = v != v ? (nan_high ? 0xFFFFFFFFu : 0u) : orderable(v);
  return (((u64)o) << 32) | (u64)(0xFFFFFFFFu - (unsigned)qi);
}

// How many of a line's nnz non-zero values SLIM ElasticNet keeps: min(nnz - 1, K), SLIMElasticNetRecommender.py:103
__device__ __forceinline__ int drop_last_keep(int K, int nnz) { return max(0, min(K, nnz - 1)); }

// What the select needs of a key type: its width, the digit nb bits wide at bit sh, the test against the prefix fixed so
// far, and fixing one more digit of the prefix.
template <typename Key> struct KeyBits;
template <> struct KeyBits<u64> {
  static constexpr int BITS = 64;
  static __device__ __forceinline__ u64 make(unsigned hi, unsigned lo) { return ((u64)hi << 32) | lo; }
  static __device__ __forceinline__ unsigned low(u64 k) { return (unsigned)k; }
  static __device__ __forceinline__ int digit(u64 k, int sh, int nb) { return (int)((k >> sh) & ((1u << nb) - 1)); }
  static __device__ __forceinline__ bool matches(u64 k, u64 prefix, u64 mask) { return (k & mask) == prefix; }
  static __device__ __forceinline__ void fix_digit(u64& prefix, u64& mask, int d, int sh, int nb) {
    prefix |= ((u64)d) << sh;
    mask |= ((u64)((1u << nb) - 1)) << sh;
  }
  static __device__ __forceinline__ bool greater(u64 a, u64 b) { return a > b; }
  static __device__ __forceinline__ bool at_least(u64 a, u64 b) { return a >= b; }
};
// 96 bits: a 64-bit ordered value (fp64), then the 32-bit tie-break.  A digit may straddle the two words.
struct Key96 {
  u64 hi;
  unsigned lo;
};
template <> struct KeyBits<Key96> {
  static constexpr int BITS = 96;
  static __device__ __forceinline__ Key96 make(u64 hi, unsigned lo) { return Key96{hi, lo}; }
  static __device__ __forceinline__ unsigned low(const Key96& k) { return k.lo; }
  static __device__ __forceinline__ int digit(const Key96& k, int sh, int nb) {
    const u64 w = sh >= 32 ? k.hi >> (sh - 32) : (k.hi << (32 - sh)) | (u64)(k.lo >> sh);
    return (int)(w & ((1u << nb) - 1));
  }
  static __device__ __forceinline__ bool matches(const Key96& k, const Key96& prefix, const Key96& mask) {
    return (k.hi & mask.hi) == prefix.hi && (k.lo & mask.lo) == prefix.lo;
  }
  static __device__ __forceinline__ void fix_digit(Key96& prefix, Key96& mask, int d, int sh, int nb) {
    const u64 m = (1u << nb) - 1;
    if (sh >= 32) {
      prefix.hi |= (u64)d << (sh - 32);
      mask.hi |= m << (sh - 32);
    } else {
      prefix.hi |= (u64)d >> (32 - sh);
      mask.hi |= m >> (32 - sh);
      prefix.lo |= (unsigned)((u64)d << sh);
      mask.lo |= (unsigned)(m << sh);
    }
  }
  static __device__ __forceinline__ bool greater(const Key96& a, const Key96& b) {
    return a.hi > b.hi || (a.hi == b.hi && a.lo > b.lo);
  }
  static __device__ __forceinline__ bool at_least(const Key96& a, const Key96& b) {
    return a.hi > b.hi || (a.hi == b.hi && a.lo >= b.lo);
  }
};

__device__ __forceinline__ void warp_or_and(u64& o, u64& a) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { o |= __shfl_xor_sync(0xffffffffu, o, off); a &= __shfl_xor_sync(0xffffffffu, a, off); }
}

// The groups that select together.  Both scan the histogram with one warp; they differ in how the scanning warp's
// result reaches the others.
//
// One warp alone, with its own histogram of 2^digit ints (16-byte aligned: the scan reads it as int4).
struct WarpSelect {
  static constexpr int SIZE = 32;
  int* hist;
  __device__ __forceinline__ bool scans() const { return true; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ void or_and(u64& o, u64& a) const { warp_or_and(o, a); }
  // the one lane that found the bin (digit >= 0) hands its values to the others
  __device__ __forceinline__ void pick(int& digit, int& need, int& bincnt) const {
    const int src = __ffs(__ballot_sync(0xffffffffu, digit >= 0)) - 1;
    digit = __shfl_sync(0xffffffffu, digit, src);
    need = __shfl_sync(0xffffffffu, need, src);
    bincnt = __shfl_sync(0xffffffffu, bincnt, src);
    __syncwarp();  // every lane has read the histogram before the next pass clears it
  }
};

// A whole CTA of THREADS (a power of two) threads; warp 0 scans the bins and passes the result through shared memory.
template <int BINS>
struct CtaSelectSmem {
  union {
    alignas(16) int hist[BINS];
    unsigned bits[4];  // the OR and the AND of all keys as 32-bit halves, before the first pass
  };
  int digit, need, bincnt;
};
template <int THREADS, int BINS>
struct CtaSelect {
  static constexpr int SIZE = THREADS;
  CtaSelectSmem<BINS>* s;
  int* hist;
  __device__ __forceinline__ explicit CtaSelect(CtaSelectSmem<BINS>& sm) : s(&sm), hist(sm.hist) {}
  __device__ __forceinline__ bool scans() const { return threadIdx.x < 32; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
  __device__ __forceinline__ void or_and(u64& o, u64& a) const {
    if (threadIdx.x == 0) { s->bits[0] = s->bits[1] = 0u; s->bits[2] = s->bits[3] = ~0u; }
    __syncthreads();
    warp_or_and(o, a);
    if ((threadIdx.x & 31) == 0) {
      atomicOr(&s->bits[0], (unsigned)o); atomicOr(&s->bits[1], (unsigned)(o >> 32));
      atomicAnd(&s->bits[2], (unsigned)a); atomicAnd(&s->bits[3], (unsigned)(a >> 32));
    }
    __syncthreads();
    o = ((u64)s->bits[1] << 32) | s->bits[0];
    a = ((u64)s->bits[3] << 32) | s->bits[2];
    __syncthreads();  // every thread has read them before the first pass clears the histogram
  }
  __device__ __forceinline__ void pick(int& digit, int& need, int& bincnt) const {
    if (digit >= 0) { s->digit = digit; s->need = need; s->bincnt = bincnt; }
    __syncthreads();
    digit = s->digit;
    need = s->need;
    bincnt = s->bincnt;
  }
};

template <typename Key>
struct Threshold {
  Key thr;   // exactly the K largest keys are >= thr
  int need;  // how many of the keys equal to thr are among them (more than one only when keys repeat); after a stop on a
             // whole bin, the size of that bin: at least the number of keys equal to thr
};

// The K-th largest of the keys at positions [0, n): key_at(q, key) sets the key of position q and returns true, or
// returns false when position q holds none.  0 < K <= the number of keys.  Called by every thread of the group.
// DIGIT: 8 or 11 bits.  SKIP (64-bit keys): one OR / AND pass first, to start below the leading digits that every key
// shares; worth it when key_at is a shared-memory read.
template <typename Key, int DIGIT, bool SKIP, class Group, class KeyAt>
__device__ __forceinline__ Threshold<Key> radix_select(const Group& g, int n, int K, KeyAt key_at) {
  typedef KeyBits<Key> KB;
  constexpr int BINS = 1 << DIGIT, PER = BINS / 32;
  const int rank = threadIdx.x & (Group::SIZE - 1);  // in the group
  static_assert(!SKIP || KB::BITS == 64, "the prefix skip is written for 64-bit keys");
  Key prefix{}, mask{};
  int shift = KB::BITS - DIGIT;  // the top digit; the lowest one is narrower when DIGIT does not divide the width
  if constexpr (SKIP) {
    u64 o = 0ull, a = ~0ull;
    for (int q = rank; q < n; q += Group::SIZE) {
      Key k;
      if (key_at(q, k)) { o |= k; a &= k; }
    }
    g.or_and(o, a);
    const u64 diff = o ^ a;
    const int hb = diff ? 63 - __clzll((long long)diff) : 0;  // the highest bit in which two keys differ
    shift = KB::BITS - DIGIT * ((KB::BITS - 1 - hb) / DIGIT + 1);
    if (shift + DIGIT < 64) {
      mask = ~0ull << (shift + DIGIT);
      prefix = o & mask;
    }
  }
  int need = K;
  // A literal 1 makes ptxas emit the warp-aggregated ATOMS.POPC.INC, meant for warps whose keys share a bin, as they do in
  // the leading passes without the skip.  After the skip the keys spread over the bins; the K-1D kernel, the only caller
  // that skips, was tuned with the plain ATOMS.ADD that a run-time 1 keeps.
  const int one = SKIP ? (n > 0 ? 1 : 0) : 1;
  for (;; shift -= DIGIT) {
    const int sh = max(shift, 0), nb = DIGIT + min(shift, 0);
    for (int b = rank; b < BINS; b += Group::SIZE) g.hist[b] = 0;
    g.sync();
    for (int q = rank; q < n; q += Group::SIZE) {
      Key k;
      if (key_at(q, k) && KB::matches(k, prefix, mask)) atomicAdd(&g.hist[KB::digit(k, sh, nb)], one);
    }
    g.sync();
    int digit = -1, rest = 0, bincnt = 0;
    if (g.scans()) {
      // lane l owns bins base .. base + PER - 1, the highest bins in lane 0, read as 16-byte vectors.  With 11-bit digits a
      // lane's 16 vectors are read 4 and 8 at a time: the unroll factors that keep topk_lines_kernel within the registers
      // of its occupancy (see there)
      const int lane = threadIdx.x & 31, base = BINS - (lane + 1) * PER;
      const int4* h = reinterpret_cast<const int4*>(g.hist + base);
      int local = 0;
#pragma unroll (PER > 8 ? 4 : PER / 4)
      for (int v = 0; v < PER / 4; ++v) {
        const int4 c = h[v];
        local += c.x + c.y + c.z + c.w;
      }
      int cum = local;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, cum, off);
        if (lane >= off) cum += t;
      }
      cum -= local;  // keys in higher bins
#pragma unroll (PER > 8 ? 8 : PER / 4)
      for (int v = PER / 4 - 1; v >= 0; --v) {
        const int4 c4 = h[v];
        const int c[4] = {c4.w, c4.z, c4.y, c4.x};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (cum < need && cum + c[e] >= need) {
            digit = base + 4 * v + 3 - e;
            rest = need - cum;
            if (PER <= 8) bincnt = c[e];
          }
          cum += c[e];
        }
      }
    }
    if (PER > 8 && digit >= 0) bincnt = g.hist[digit];  // one register less in the loop: topk_lines_kernel's occupancy
    g.pick(digit, rest, bincnt);
    KB::fix_digit(prefix, mask, digit, sh, nb);
    need = rest;
    if (bincnt == need || shift <= 0) break;
  }
  return Threshold<Key>{prefix, need};
}

}  // namespace b200
