// K1-D: the binary similarity kernel for large catalogues with sparse co-occurrence counts (included by sim_topk.cu inside
// namespace b200::sim).  Replaces Compute_Similarity_Cython.pyx:327-408 (gather / accumulate) and :467-568 (normalise,
// top-K, emit) for every-stored-value-is-1 data, like the window kernel, with a different on-chip representation.
//
// What per-phase cycle counters of the two earlier kernels showed:
//   window kernel (16-bit counters, 2 windows of 200 KB): a latency-bound gather (CSC entry -> row bounds -> row, two
//     dependent trips to memory) and more time sweeping / selecting over 2 x 100 K cells;
//   bitmap kernel K1-C (three thermometer bitmaps, TMA ring): shared-memory atomics that RETURN a value run at about one
//     per cycle per SM, and it ran a radix select per level.
// So: counters must be bumped with fire-and-forget atomics, the gather needs one dependent trip and many rows in flight,
// and the per-column passes must touch few bytes.
//
// Representation.  4-bit counters, eight per 32-bit word: 200 K neighbours = 100 KB, ONE pass per column, and two CTAs
// (512 threads each) per SM, so one CTA's selection overlaps the other's gather.  A counter that would reach 16 carries
// into its neighbour -- silently, but not undetectably: a carry lowers the sum of all nibbles by 15 (by 16 out of a word),
// never raises it, so  "sum of nibbles == number of increments" holds iff no counter overflowed.  The sweep that looks for
// candidates computes that sum anyway; a column that fails the check is handed to the window kernel (redo list), as are the
// columns the host routes there directly (dense co-occurrence).  Exactness is unchanged.
//
// What bounds it: the ~50 K shared-memory atomics of a C5 column issue slowly when both CTAs of an SM gather at once, and
// nothing overlaps them with the sweep / select / emit that follow: the two CTAs fall into lockstep.
// Tried and left out: a bank-spread accumulator (word = (j >> 8) << 5 | j & 31 with rows re-sorted by bank:
// average bank crowding 3.1 -> 2.0 in simulation) changed nothing, so bank conflicts are not the limit; L2 prefetches of the
// next column's rows and pre-loaded row locations changed nothing either; a per-SM token that lets one CTA gather at a time
// showed that ONE CTA's gather alone takes as long (latency-bound with 16 warps x 4 rows in flight), so anti-phase
// buys nothing; replacing the returning atomics of the candidate collection by a two-pass sweep with prefix sums only moved
// time from the sweep into the second pass, and an atomic-free one-pass sweep (per-warp candidate regions, shuffle prefix
// sums, two vectors in flight) did not shorten the sweep: its shared loads queue behind the OTHER CTA's atomics.  What would: more CTAs per SM in different phases (two neighbour windows of
// 50 KB counters each: 3-4 CTAs) or two accumulators per CTA with warp-specialised gather / select.
//
// Gather.  The CSC side stores, per entry, where the user's padded row lives (csc_seg: start and length in 16-byte
// chunks), so a warp reads 32 of them with one coalesced load and then streams those rows with 128-bit loads, four rows in
// flight per warp: 32 warps x 4 rows x ~400 B = 50 KB in flight per SM against a bandwidth-delay product of ~18 KB.
//
// Selection.  The neighbour axis is numbered by ascending norm term, and every formula served here increases with the
// count and decreases with the neighbour's norm term.  One sweep finds the cells with count >= 3 (bit tricks on whole
// words), they are evaluated exactly into 64-bit keys (similarity bits << 32 | ~original index: ties -> ascending index).
// If there are at least K of them, the similarity of (count 3, largest norm) is a floor of the K-th best, and count-2 /
// count-1 cells can only matter in the leading norm tiles whose best possible similarity reaches the floor (none at C5).
// One radix select (8-bit digits, 512 threads) at the end keeps the K best.  Pushes are chunked by norm tile with known
// cell counts, so the key buffer cannot overflow; a full buffer is pruned to the K best first (raising the floor).

constexpr int D_THREADS = 512;
constexpr int D_WARPS = D_THREADS / 32;
constexpr int D_ROWS = 4;        // rows in flight per warp
constexpr int D_TILE_LOG2 = 10;  // norm tile: 1024 neighbours = 128 counter words

struct K1DShared {
  int item, nbuf, cnt, adds, nibsum, tstop, chunk_end, chunk_cnt;
  int need, digit, bincnt, ncand, expect;
  u64 kor, kand;
  int hist[256];
};

// bit 0 of every nibble of the result is set iff that nibble of w is >= 3 / == 2 / == 1
__device__ __forceinline__ unsigned nib_ge3(unsigned w) { return (((w | (w >> 1)) >> 2) | (w & (w >> 1))) & 0x11111111u; }
__device__ __forceinline__ unsigned nib_eq2(unsigned w) { return (w >> 1) & ~w & ~(w >> 2) & ~(w >> 3) & 0x11111111u; }
__device__ __forceinline__ unsigned nib_eq1(unsigned w) { return w & ~(w >> 1) & ~(w >> 2) & ~(w >> 3) & 0x11111111u; }
__device__ __forceinline__ unsigned nib_level(unsigned w, int level) {
  return level >= 3 ? nib_ge3(w) : (level == 2 ? nib_eq2(w) : nib_eq1(w));
}
__device__ __forceinline__ int nib_sum(unsigned w) {
  const unsigned b = (w & 0x0F0F0F0Fu) + ((w >> 4) & 0x0F0F0F0Fu);
  return (int)__dp4a(b, 0x01010101u, 0u);
}

// Block-wide (all D_THREADS threads): keeps the K largest keys of buf[0..n) compacted at the front (any order), returns
// the K-th largest key (0 when n <= K: nothing is cut).  Keys are distinct and non-zero.  MSB-first radix select with
// 8-bit digits; stops as soon as a whole bin is taken.
__device__ u64 d_select(u64* buf, int n, int K, K1DShared* ds, int* n_out) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (n <= K) { *n_out = n; return 0ull; }
  // digits above the highest bit in which two keys differ are the same for every key: start below them
  {
    if (tid == 0) { ds->kor = 0ull; ds->kand = ~0ull; }
    __syncthreads();
    u64 o = 0ull, a = ~0ull;
    for (int q = tid; q < n; q += D_THREADS) { const u64 k = buf[q]; o |= k; a &= k; }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { o |= __shfl_xor_sync(0xffffffffu, o, off); a &= __shfl_xor_sync(0xffffffffu, a, off); }
    if ((tid & 31) == 0) { atomicOr(&ds->kor, o); atomicAnd(&ds->kand, a); }
    __syncthreads();
  }
  const u64 diff = ds->kor ^ ds->kand;
  int pass = diff ? (63 - __clzll((long long)diff)) >> 3 : 0;
  u64 prefix = pass < 7 ? (ds->kor >> ((pass + 1) * 8)) << ((pass + 1) * 8) : 0ull;
  int need = K;
  const int one = n > 0 ? 1 : 0;  // a run-time 1: a literal makes ptxas emit ATOMS.POPC.INC inside a loop that peels one address per trip
  for (; pass >= 0; --pass) {
    const int shift = pass * 8;
    if (tid < 256) ds->hist[tid] = 0;
    __syncthreads();
    for (int q = tid; q < n; q += D_THREADS) {
      const u64 k = buf[q];
      if (pass == 7 || (k >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&ds->hist[(int)((k >> shift) & 255ull)], one);
    }
    __syncthreads();
    if (tid < 32) {  // one warp: bins 255 .. 0, eight per lane, highest bins in lane 0
      int c[8], local = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) { c[b] = ds->hist[255 - (tid * 8 + b)]; local += c[b]; }
      int incl = local;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (tid >= off) incl += t;
      }
      int cum = incl - local;  // keys in higher bins
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (cum < need && cum + c[b] >= need) { ds->digit = 255 - (tid * 8 + b); ds->need = need - cum; ds->bincnt = c[b]; }
        cum += c[b];
      }
    }
    __syncthreads();
    prefix |= ((u64)ds->digit) << shift;
    need = ds->need;
    const int bincnt = ds->bincnt;
    __syncthreads();
    if (bincnt == need) break;  // the whole bin survives: every key with this prefix is kept
  }
  const u64 thr = prefix;  // undecided low digits are zero: the smallest key the kept bins can hold
  // compaction through registers (n <= 8 * D_THREADS is guaranteed by the host-side cap)
  u64 keep[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int i = q * D_THREADS + tid;
    const u64 k = i < n ? buf[i] : 0ull;
    keep[q] = k >= thr ? k : 0ull;
  }
  if (tid == 0) ds->cnt = 0;
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 8; ++q)
    if (keep[q]) buf[atomicAdd(&ds->cnt, 1)] = keep[q];
  __syncthreads();
  *n_out = ds->cnt;
  return thr;
}

template <int F>
__global__ void __launch_bounds__(D_THREADS, 2) sim_k1d_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ K1DShared ds;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = p.bm_words;                   // allocated counter words (multiple of 4)
  const int Wr = (p.n_cols + 7) >> 3;         // words that hold real neighbours
  const int ntile = p.ntile;
  unsigned* acc = reinterpret_cast<unsigned*>(smem_raw);
  u64* buf = reinterpret_cast<u64*>(smem_raw + (size_t)W * 4);
  float* tbs = reinterpret_cast<float*>(buf + p.cap_d);
  int* tcnt = reinterpret_cast<int*>(tbs + ntile + 1);

  for (int i = tid; i < W; i += D_THREADS) acc[i] = 0u;
  for (int i = tid; i <= ntile; i += D_THREADS) tbs[i] = p.tbnd[i];
  for (int i = tid; i < ntile; i += D_THREADS) tcnt[i] = 0;
  long long prof_t = p.prof ? clock64() : 0;
  const int K = p.K;

  for (;;) {
    __syncthreads();
    if (tid == 0) { ds.item = atomicAdd(p.counter, 1); ds.nbuf = 0; ds.adds = 0; ds.nibsum = 0; ds.ncand = 0; }
    __syncthreads();
    const int item = ds.item;
    if (item >= p.n_range) break;
    const int4 wi = __ldg(p.worklist + item);
    const int col = wi.x, lc = wi.y, cs = wi.z, ce = wi.w;
    const size_t out_base = (size_t)lc * K;
    const float Ai = p.A[col];

    // ---------------- gather: one fire-and-forget shared atomic per gathered entry, nothing else per entry
    int expect = 0;  // increments this warp's rows must produce: per row 4 * chunks - padding - 1 (the diagonal, pyx:396)
    for (int k0 = cs + warp * 32; k0 < ce; k0 += D_WARPS * 32) {
      const int nrows = min(32, ce - k0);
      int2 seg = make_int2(0, 0);
      if (lane < nrows) {
        seg = __ldg(p.csc_seg + k0 + lane);
        expect += 4 * (seg.y >> 2) - (seg.y & 3) - 1;
      }
      for (int r0 = 0; r0 < nrows; r0 += D_ROWS) {
        int4 v[D_ROWS];
        int rs[D_ROWS], rn[D_ROWS];
#pragma unroll
        for (int q = 0; q < D_ROWS; ++q) {
          const int r = r0 + q;
          rs[q] = __shfl_sync(0xffffffffu, seg.x, r & 31);
          rn[q] = r < nrows ? (__shfl_sync(0xffffffffu, seg.y, r & 31) >> 2) : 0;
          if (lane < rn[q]) v[q] = __ldg(reinterpret_cast<const int4*>(p.csr_idx1) + (size_t)rs[q] + lane);
        }
#pragma unroll
        for (int q = 0; q < D_ROWS; ++q) {
          int c0 = 0;
          for (;;) {
            if (c0 + lane < rn[q]) {
              const int jj[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const int j = jj[c];
                if ((unsigned)j < (unsigned)p.n_cols && j != col) atomicAdd(&acc[j >> 3], 1u << ((j & 7) << 2));
              }
            }
            c0 += 32;
            if (c0 >= rn[q]) break;  // rows longer than 32 chunks (128 entries): next 512 bytes
            if (c0 + lane < rn[q]) v[q] = __ldg(reinterpret_cast<const int4*>(p.csr_idx1) + (size_t)rs[q] + c0 + lane);
          }
        }
      }
    }
    expect = __reduce_add_sync(0xffffffffu, expect);
    if (lane == 0 && expect) atomicAdd(&ds.adds, expect);
    __syncthreads();
    PROF_MARK(1);

    // ---------------- one sweep (128-bit loads): nibble checksum, cells with count >= 3 per norm tile, and the cells themselves
    // as packed (neighbour << 4 | count) candidates while they fit the key buffer
    {
      int ns = 0;
      unsigned* cand = reinterpret_cast<unsigned*>(buf);
      const int cand_cap = p.cap_d;
      const uint4* acc4 = reinterpret_cast<const uint4*>(acc);
      for (int i4 = tid; i4 < ((Wr + 3) >> 2); i4 += D_THREADS) {
        const uint4 w4 = acc4[i4];
        if (!(w4.x | w4.y | w4.z | w4.w)) continue;
        const unsigned ww[4] = {w4.x, w4.y, w4.z, w4.w};
        unsigned bytes = 0u, any = 0u, m[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          bytes += (ww[e] & 0x0F0F0F0Fu) + ((ww[e] >> 4) & 0x0F0F0F0Fu);  // every byte <= 4 * 30
          m[e] = nib_ge3(ww[e]);
          any |= m[e];
        }
        ns += (int)__dp4a(bytes, 0x01010101u, 0u);
        if (any) {
          const int c3 = __popc(m[0]) + __popc(m[1]) + __popc(m[2]) + __popc(m[3]);
          atomicAdd(&tcnt[(i4 * 4) >> (D_TILE_LOG2 - 3)], c3);  // the four words of a vector lie in one tile
          int pos = atomicAdd(&ds.ncand, c3);
          if (pos + c3 <= cand_cap) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              unsigned mm = m[e];
              while (mm) {
                const int q = (__ffs(mm) - 1) >> 2;
                mm &= mm - 1;
                cand[pos++] = ((unsigned)((i4 * 4 + e) * 8 + q) << 4) | ((ww[e] >> (q << 2)) & 15u);
              }
            }
          }
        }
      }
      ns = __reduce_add_sync(0xffffffffu, ns);
      if (lane == 0 && ns) atomicAdd(&ds.nibsum, ns);
    }
    __syncthreads();
    const bool forced = p.fail_every > 0 && (lc % p.fail_every) == 0;  // test hook: exercises the redo path
    if (ds.nibsum != ds.adds || forced) {
      // a counter overflowed: the window kernel redoes this column; leave clean state behind
      __syncthreads();
      if (tid == 0) p.redo[atomicAdd(p.fail, 1)] = lc;
      for (int i = tid; i < (W >> 2); i += D_THREADS) reinterpret_cast<int4*>(acc)[i] = make_int4(0, 0, 0, 0);
      for (int i = tid; i < ntile; i += D_THREADS) tcnt[i] = 0;
      continue;
    }
    PROF_MARK(2);

    u64 thr = 0ull;  // keys below it cannot be among the K best
    int n_have = 0;  // block-uniform copy of ds.nbuf between pushes
    const int n3 = ds.ncand;
    const bool collected = n3 <= p.cap_d;  // every count >= 3 cell sits in the buffer as a packed candidate
    if (collected) {
      // all candidates at once: the norm-term gathers of a column are one round trip, not one per sweep step
      const unsigned* cand = reinterpret_cast<const unsigned*>(buf);
      u64 keys[4];  // cap_d <= 4 * D_THREADS on this path (host)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int t = q * D_THREADS + tid;
        keys[q] = 0ull;
        if (t < n3) {
          const unsigned cd = cand[t];
          const int2 bn = __ldg(p.BN + (cd >> 4));
          const float sv = sim_value<F>(p, (float)(cd & 15u), Ai, __int_as_float(bn.x));
          if (sv > 0.f) keys[q] = (((u64)__float_as_uint(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn.y);
        }
      }
      __syncthreads();  // every packed candidate has been read: the keys may overwrite them
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (keys[q]) buf[atomicAdd(&ds.nbuf, 1)] = keys[q];
      for (int i = tid; i < ntile; i += D_THREADS) tcnt[i] = 0;
      __syncthreads();
      n_have = ds.nbuf;
      if (n_have >= K) {
        // every key has count >= 3 and a norm term <= the largest one: that similarity is a floor of the K-th best
        const float fl = sim_value<F>(p, 3.f, Ai, tbs[ntile]) * (1.f - 1e-6f);
        if (fl > 0.f) thr = ((u64)__float_as_uint(fl)) << 32;
      }
      PROF_MARK(3);
    }
#pragma unroll 1
    for (int level = collected ? 2 : 3; level >= 1; --level) {
      int t_end = ntile;
      if (level < 3) {
        // exactly-`level` cells reach the floor only in the leading norm tiles (tbs[t] = smallest norm term of tile t)
        if (thr == 0ull) {
          t_end = ntile;  // no floor yet: fewer than K candidates so far, every cell counts
        } else {
          const float tsim = __uint_as_float((unsigned)(thr >> 32));
          if (tid == 0) ds.tstop = ntile;
          __syncthreads();
          for (int t = tid; t < ntile; t += D_THREADS)
            if (!(sim_value<F>(p, (float)level, Ai, tbs[t]) >= tsim)) atomicMin(&ds.tstop, t);
          __syncthreads();
          t_end = ds.tstop;
          __syncthreads();  // everyone has read it before thread 0 of the next level resets it
        }
        if (t_end == 0) continue;
        // cells of this level per allowed tile
        const int w_end = min(Wr, t_end << (D_TILE_LOG2 - 3));
        for (int i = tid; i < w_end; i += D_THREADS) {
          const unsigned w = acc[i];
          if (!w) continue;
          const int c = __popc(nib_level(w, level));
          if (c) atomicAdd(&tcnt[i >> (D_TILE_LOG2 - 3)], c);
        }
        __syncthreads();
      }
      // pushes in chunks of whole tiles whose cell counts are known to fit the buffer
      int t0 = 0;
      while (t0 < t_end) {
        if (tid == 0) {
          int t1 = t0, c = 0;
          while (t1 < t_end && n_have + c + tcnt[t1] <= p.cap_d) { c += tcnt[t1]; ++t1; }
          ds.chunk_end = t1;
          ds.chunk_cnt = c;
        }
        __syncthreads();
        const int t1 = ds.chunk_end;
        if (t1 == t0) {
          // the next tile does not fit: prune to the K best (exact floor), which always makes room (cap_d >= K + 1024)
          int kept;
          const u64 t2 = d_select(buf, n_have, K, &ds, &kept);
          thr = max(thr, t2);
          if (tid == 0) ds.nbuf = kept;
          n_have = kept;
          __syncthreads();
          continue;
        }
        if (ds.chunk_cnt > 0) {
          const int w_lo = t0 << (D_TILE_LOG2 - 3), w_hi = min(Wr, t1 << (D_TILE_LOG2 - 3));
          for (int i = w_lo + tid; i < w_hi; i += D_THREADS) {
            const unsigned w = acc[i];
            if (!w) continue;
            unsigned m = nib_level(w, level);
            while (m) {
              const int q = (__ffs(m) - 1) >> 2;
              m &= m - 1;
              const int j = i * 8 + q;
              const float d = (float)((w >> (q << 2)) & 15u);
              const int2 bn = __ldg(p.BN + j);
              const float sv = sim_value<F>(p, d, Ai, __int_as_float(bn.x));
              const u64 key = (((u64)__float_as_uint(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn.y);
              if (sv > 0.f && key >= thr) buf[atomicAdd(&ds.nbuf, 1)] = key;
            }
          }
        }
        __syncthreads();
        n_have = ds.nbuf;
        t0 = t1;
      }
      for (int i = tid; i < ntile; i += D_THREADS) tcnt[i] = 0;
      __syncthreads();
      if (n_have >= K) {
        if (level == 3 && thr == 0ull) {
          // every key pushed so far has count >= 3 and a norm term <= the largest one: that similarity is a floor of the
          // K-th best (the formulas increase with the count and decrease with the norm term); no select needed
          const float fl = sim_value<F>(p, 3.f, Ai, tbs[ntile]) * (1.f - 1e-6f);
          if (fl > 0.f) thr = ((u64)__float_as_uint(fl)) << 32;
        } else if (level == 2 && n_have > K) {
          int kept;
          const u64 t2 = d_select(buf, n_have, K, &ds, &kept);  // exact floor before the widest level
          thr = max(thr, t2);
          if (tid == 0) ds.nbuf = kept;
          n_have = kept;
          __syncthreads();
        }
      }
      if (level == 3) PROF_MARK(3); else if (level == 2) PROF_MARK(4); else PROF_MARK(5);
    }

    // ---------------- the K best, emit, clear
    {
      int kept;
      d_select(buf, n_have, K, &ds, &kept);
      n_have = kept;
    }
    for (int t = tid; t < n_have; t += D_THREADS) {
      const u64 k64 = buf[t];
      emit_entry(p, out_base + t, (int)(0xFFFFFFFFu - (unsigned)k64), __uint_as_float((unsigned)(k64 >> 32)));
    }
    for (int t = n_have + tid; t < K; t += D_THREADS) {
      emit_entry(p, out_base + t, -1, 0.f);
    }
    if (tid == 0) emit_count(p, lc, n_have);
    for (int i = tid; i < (W >> 2); i += D_THREADS) reinterpret_cast<int4*>(acc)[i] = make_int4(0, 0, 0, 0);
    PROF_MARK(6);
  }
}

// tb[t] = norm term at neighbour min(t << D_TILE_LOG2, n_cols - 1), t = 0 .. ntile
__global__ void k1d_tile_bounds_kernel(const int2* __restrict__ BN, int n_cols, int ntile, float* tb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > ntile) return;
  tb[t] = __int_as_float(BN[min(t << D_TILE_LOG2, n_cols - 1)].x);
}

// csc_seg[q] = where the padded single-window row of CSC entry q's user lives: x = start in 16-byte chunks,
// y = chunks << 2 | padding entries in the last chunk (0..3)
__global__ void k1d_csc_seg_kernel(const int* __restrict__ csc_idx, const int* __restrict__ split1, const int* __restrict__ csr_ptr,
                                   long long nnz, int2* seg) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x) {
    const int u = csc_idx[q];
    const int s = split1[2 * (size_t)u], e = split1[2 * (size_t)u + 1];
    const int len = csr_ptr[u + 1] - csr_ptr[u];
    seg[q] = make_int2(s >> 2, (((e - s) >> 2) << 2) | ((e - s) - len));
  }
}
