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
// Gather.  Rows are packed seven entries to a 16-byte chunk (a 32-bit index and six 16-bit gaps: the layout is described
// above K1DShared), so a gathered entry costs 2.3 bytes instead of 4.  The CSC side stores, per entry, where the user's
// row lives (csc_seg: first chunk and chunk count), so a warp reads 32 of them with one coalesced load and then streams
// those rows with 128-bit loads, a half warp per row (~15 chunks at C5) and four loads of two rows in flight per warp:
// 32 warps x 8 rows x ~240 B = 60 KB in flight per SM.  With a whole warp per row more than half the lanes idle and the
// kernel issues nearly twice the shared-atomic instructions per entry: it was 12 % slower than with four entries per chunk.
//
// Selection.  The neighbour axis is numbered by ascending norm term, and every formula served here increases with the
// count and decreases with the neighbour's norm term.  One sweep finds the cells with count >= 3 (bit tricks on whole
// words), they are evaluated exactly into 64-bit keys (similarity bits << 32 | ~original index: ties -> ascending index).
// If there are at least K of them, the similarity of (count 3, largest norm) is a floor of the K-th best, and count-2 /
// count-1 cells can only matter in the leading norm tiles whose best possible similarity reaches the floor (none at C5).
// One radix select (select.cuh: 8-bit digits, 512 threads) at the end keeps the K best.  Pushes are chunked by norm tile
// with known cell counts, so the key buffer cannot overflow; a full buffer is pruned to the K best first (raising the
// floor).

constexpr int D_THREADS = 512;
constexpr int D_WARPS = D_THREADS / 32;
constexpr int D_ROWS = 4;        // rows in flight per warp
constexpr int D_TILE_LOG2 = 10;  // norm tile: 1024 neighbours = 128 counter words

// The K1-D row layout.  Every user's sorted row, `copies` times back to back (copies = 2: the indices, then the same
// indices + n_cols, so that the upper pass's cyclic window of an entry is one range of the row), as 16-byte chunks of up to
// seven entries: int4 {base, g1 | g2 << 16, g3 | g4 << 16, g5 | g6 << 16}.  Entry 0 is `base`, an absolute index; entry e
// is entry e - 1 plus the 16-bit gap g_e.  Rows are sorted and distinct and the second copy starts first + n_cols - last
// >= 1 after the first ends, so a real gap is >= 1: gap 0 means "no entry", and every slot after it is empty too.  An
// entry 65 536 or more after its predecessor starts a new chunk as its base (at C5 the mean gap is 2 000).  Every chunk's
// base is a real entry and the bases of a row ascend, so the chunk that holds a given entry is found by value.
constexpr int K1D_GAPS = 6;
__device__ __forceinline__ int k1d_gap(const int4& c, int e) {  // g_(e + 1)
  const int w = e < 2 ? c.y : (e < 4 ? c.z : c.w);
  return (e & 1) ? (int)((unsigned)w >> 16) : (w & 0xffff);
}

struct K1DShared {
  int item, nbuf, cnt, nibsum, tstop, chunk_end, chunk_cnt;
  int ncand, expect;
  CtaSelectSmem<256> sel;
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
// the K-th largest key (0 when n <= K: nothing is cut).  Keys are distinct and non-zero.
__device__ u64 d_select(u64* buf, int n, int K, K1DShared* ds, int* n_out) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (n <= K) { *n_out = n; return 0ull; }
  const auto sel_key = [&](int q, u64& key) {
    key = buf[q];
    return true;
  };
  const u64 thr = radix_select<u64, 8, true>(CtaSelect<D_THREADS, 256>(ds->sel), n, K, sel_key).thr;
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
  const int n_items = p.n_range_dev ? *p.n_range_dev : p.n_range;

  for (;;) {
    __syncthreads();
    if (tid == 0) { ds.item = atomicAdd(p.counter, 1); ds.nbuf = 0; ds.nibsum = 0; ds.ncand = 0; }
    __syncthreads();
    const int item = ds.item;
    if (item >= n_items) break;
    const int4 wi = __ldg(p.worklist + item);
    const int col = wi.x, lc = wi.y, cs = wi.z, ce = wi.w;
    const size_t out_base = (size_t)lc * K;
    const float Ai = p.A[col];
    const int adds = __ldg(p.col_adds + col);  // increments the column's rows must produce: per row its entries - 1 (the diagonal, pyx:396)

    // ---------------- gather: one fire-and-forget shared atomic per gathered entry, nothing else per entry
    for (int k0 = cs + warp * 32; k0 < ce; k0 += D_WARPS * 32) {
      const int nrows = min(32, ce - k0);
      int2 seg = make_int2(0, 0);
      if (lane < nrows) seg = __ldg(p.csc_seg + k0 + lane);
      // a half warp per row (a C5 row is ~15 chunks): D_ROWS loads of two rows each in flight, every lane's seven entries
      // decoded by a running sum over the gaps
      const int hl = lane & 15, hh = lane >> 4;
      for (int r0 = 0; r0 < nrows; r0 += 2 * D_ROWS) {
        int4 v[D_ROWS];
        int rs[D_ROWS], rn[D_ROWS];
#pragma unroll
        for (int q = 0; q < D_ROWS; ++q) {
          const int r = r0 + 2 * q + hh;
          rs[q] = __shfl_sync(0xffffffffu, seg.x, r & 31);
          rn[q] = __shfl_sync(0xffffffffu, seg.y, r & 31);
          if (r >= nrows) rn[q] = 0;
          if (hl < rn[q]) v[q] = __ldg(p.csr_idx1 + (size_t)rs[q] + hl);
        }
#pragma unroll
        for (int q = 0; q < D_ROWS; ++q) {
          int c0 = 0;
          for (;;) {
            if (c0 + hl < rn[q]) {
              // the last chunk of the first copy can run on into the second one: j < n_cols masks those entries
              int j = v[q].x;
              if (j < p.n_cols && j != col) atomicAdd(&acc[j >> 3], 1u << ((j & 7) << 2));
#pragma unroll
              for (int e = 0; e < K1D_GAPS; ++e) {
                const int g = k1d_gap(v[q], e);
                j += g;
                if (g && j < p.n_cols && j != col) atomicAdd(&acc[j >> 3], 1u << ((j & 7) << 2));
              }
            }
            c0 += 16;
            if (c0 >= rn[q]) break;  // rows longer than 16 chunks (up to 112 entries): next 256 bytes
            if (c0 + hl < rn[q]) v[q] = __ldg(p.csr_idx1 + (size_t)rs[q] + c0 + hl);
          }
        }
      }
    }
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
    if (ds.nibsum != adds || forced) {
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

// ---------------------------------------------------------------------------------------------------------------------
// Pair path: every co-occurrence count C[i][j] = C[j][i] is gathered once.
//
// The kernel above builds C[i][j] in pass i and again in pass j: it streams the whole row of every user of column i.  On a
// call that covers every column, the upper pass counts each pair once, in a cyclic half window: pass i counts neighbour j
// iff d = (j - i) mod n lies in [1, h], h = (n - 1) / 2, and, when n is even, the antipodal d = n / 2 for i < n / 2 only
// (k1d_window_size).  Half the gathered entries and half the shared atomics, and -- unlike the j > i split, which gives
// column 0 every neighbour and the last column none -- every pass needs at most n / 2 counters and gathers about half of
// each of its rows.  Each user's row is stored twice, back to back (the indices, then the same indices + n), so that the
// window of a CSC entry is one range of the doubled row.  It writes column
// i's cells with count >= 3 as one contiguous own list and counts them into deg[j]; the exchange copies each cell into the
// mirror list of j, so column c's candidates are its own list plus its mirror list, and the select kernel (one warp per
// column) applies the rule of the kernel above to them: with at least K positive keys
// and no count-2 / count-1 cell that can reach the floor sim(3, largest norm term) (bounded by the smallest norm term of
// the columns with at least 2 / 1 users), the K best count >= 3 cells are the answer -- the same keys from the same counts
// and norm terms, so the output is the same.  Every other column (fewer
// than K candidates, count-2 / count-1 cells that matter, more candidates than the handle's sel_cap) is appended to a device
// redo list that the kernel above then computes in full.  A counter overflow in the upper pass (the nibble checksum over
// the window increments) or a full list sets a flag on the device, and the select kernel then hands EVERY column to
// the kernel above: exactness never depends on the pair path.  Whether a handle takes the path at all is decided at create
// time from the norm terms and the column lengths (k1d_pair_gate in sim_topk.cu): a column handed back costs a full pass
// on top of the upper pass, so the path only pays when the select kernel can decide nearly every column.

// Launch shape of the upper pass: U_CTAS CTAs of U_THREADS threads per SM (half-window counters: 50 KB at 200 K columns),
// so that several columns per SM are in different phases, and loads of 32 chunks issued U_STEPS at a time per warp, double
// buffered: the next U_STEPS are in flight while the current ones are counted.  The -D overrides are for A/B builds
// (tools/build_variant.py).
#ifndef B200_U_THREADS
#define B200_U_THREADS 256
#endif
#ifndef B200_U_CTAS
#define B200_U_CTAS 4
#endif
#ifndef B200_U_STEPS
#define B200_U_STEPS 3
#endif
#ifndef B200_U_STAGE
#define B200_U_STAGE 1024
#endif
constexpr int U_THREADS = B200_U_THREADS;
constexpr int U_WARPS = U_THREADS / 32;
constexpr int U_CTAS = B200_U_CTAS;
constexpr int U_STEPS = B200_U_STEPS;
constexpr int U_STAGE = B200_U_STAGE;  // count >= 3 cells of one column staged in shared memory before one global reservation

// cells of pass c's window (see above); at most n / 2
__host__ __device__ __forceinline__ int k1d_window_size(int n, int c) { return ((n - 1) >> 1) + ((n & 1) == 0 && c < (n >> 1) ? 1 : 0); }
// counter words of the upper pass: every window, rounded to whole 16-byte vectors
__host__ __device__ __forceinline__ int k1d_upper_words(int n) { return (((n >> 1) + 7) / 8 + 3) / 4 * 4; }
// own_n flag: the column's cells overflowed its stage; the cells past it went to the loose list, so its own list is
// incomplete and the select kernel hands the column to the redo list
constexpr int OWN_SPILLED = (int)0x80000000u;

struct K1DUpShared {
  int item, nibsum, ncand, nst;
  int4 wi;  // worklist_up[item], fetched by thread 0 while the previous column was counted
  unsigned long long base;
};

// One gathered entry: cell t of the window is counted iff `ok`.  Counting is straight-line code: every entry issues one
// fire-and-forget shared reduction on a 32-bit shared address (acc_s: the counters' base in the shared window), and an
// entry that does not count adds 0 to word `lane` (distinct banks, inside acc + stage: U_STAGE >= 32).  Not a predicated
// reduction: ptxas turns that back into a branch region per entry (BSSY / BRA / BSYNC) with the address math inside.
static_assert(U_STAGE >= 32, "an entry that does not count adds 0 to shared word `lane`");
__device__ __forceinline__ void k1d_up_count(unsigned acc_s, int lane, unsigned t, bool ok) {
  // word t / 8, nibble t % 8: 1 << ((t << 2) & 31), the wrap of the funnel shift
  const unsigned word = ok ? t >> 3 : (unsigned)lane, inc = ok ? __funnelshift_l(0u, 1u, t << 2) : 0u;
  asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(acc_s + (word << 2)), "r"(inc) : "memory");
}

__global__ void __launch_bounds__(U_THREADS, U_CTAS) sim_k1d_upper_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ K1DUpShared us;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = p.n_cols;
  const int W = k1d_upper_words(n);
  unsigned* acc = reinterpret_cast<unsigned*>(smem_raw);
  unsigned* stage = acc + W;
  const unsigned acc_s = (unsigned)__cvta_generic_to_shared(acc);
  for (int i = tid; i < W; i += U_THREADS) acc[i] = 0u;
  if (blockIdx.x == 0 && tid == 0 && p.fail_every > 0) atomicExch(p.pair_fail, 1);  // test hook: exercises the fallback
  long long prof_t = p.prof ? clock64() : 0;
  // Work items are taken one column ahead: thread 0 takes the next one (and reads the fallback flag alongside) while the
  // current column gathers, and loads its work item before the sweep, so a column starts with its descriptor loads.  Once
  // the call has fallen back, the remaining columns are not worth gathering: the CTA stops.
  if (tid == 0) {
    const int it = atomicAdd(p.counter, 1);
    us.item = *(volatile int*)p.pair_fail ? p.n_range : it;
    if (us.item < p.n_range) us.wi = __ldg(p.worklist_up + us.item);
    us.nibsum = 0; us.ncand = 0; us.nst = 0;
  }
  __syncthreads();

  for (;;) {
    // us.item / us.wi: written by thread 0 before a barrier (the one above, or the previous column's sweep barrier), and
    // rewritten only after this column's gather barrier
    const int item = us.item;
    if (item >= p.n_range) break;
    const int4 wi = us.wi;
    const int col = wi.x, adds = wi.y, cs = wi.z, ce = wi.w;  // adds: the increments of the column's windows
    const int size_c = k1d_window_size(n, col);
    int it_next = 0, failed = 0;
    if (tid == 0) {
      it_next = atomicAdd(p.counter, 1);
      failed = *(volatile int*)p.pair_fail;
    }

    // ---------------- gather over the row windows: cell t = j' - col - 1 of doubled-row index j', counted iff t < size_c,
    // which masks the entries of the first and last chunk outside the window; a gap of 0 is padding.  A window is half a
    // row on average (C5: ~8 chunks), so one row per warp load would leave most lanes idle and issue as many
    // loads and atomic instructions as the whole row; instead the 32 windows of a batch are one stream of chunks, every
    // lane of every load busy.  Rows with chunks sit compacted in the low lanes; lane r holds row r's [beg, end) in the
    // stream, and the row of stream position f is the number of rows that end at or before f.  A warp's batches are one
    // pipeline: the loads of its next U_STEPS steps (and the descriptors of its next batch) are in flight while it counts
    // the current ones.  A position past the batch's stream loads nothing and decodes as {col, no gaps}: t = -1, never
    // counted.
    {
      const unsigned sz = (unsigned)size_c;
      int k0 = cs + warp * 32;
      const auto desc = [&](int k) {
        int2 s = make_int2(0, 0);
        if (k + lane < ce) s = __ldg(p.csc_win + k + lane);
        return s;
      };
      int rstart = 0, beg = 0, end = 0, nr = 0, total = 0, b0 = 0;  // the open batch, and its next stream position
      const auto open = [&](int2 seg) {
        const unsigned nz = __ballot_sync(0xffffffffu, seg.y > 0);
        nr = __popc(nz);
        const int src = lane < nr ? (int)__fns(nz, 0, lane + 1) : 0;
        rstart = __shfl_sync(0xffffffffu, seg.x, src);
        const int sy = __shfl_sync(0xffffffffu, seg.y, src);
        const int rn = lane < nr ? sy : 0;
        end = rn;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, end, off);
          if (lane >= off) end += t;
        }
        beg = end - rn;
        total = __shfl_sync(0xffffffffu, end, 31);
        b0 = 0;
      };
      bool live = k0 < ce;  // the warp has steps left to issue
      int2 seg_next = make_int2(0, 0);
      if (live) {
        const int2 seg = desc(k0);
        seg_next = desc(k0 + U_WARPS * 32);
        open(seg);
      }
      // loads the next U_STEPS steps of the stream into v, then moves on to the next batch if this one is done
      const auto issue = [&](int4 (&v)[U_STEPS]) {
#pragma unroll
        for (int q = 0; q < U_STEPS; ++q) {
          const int base = b0 + 32 * q, f = base + lane;
          const unsigned before = __ballot_sync(0xffffffffu, lane < nr && end <= base);
          const unsigned ends = __reduce_or_sync(0xffffffffu, (lane < nr && end > base && end - base < 32) ? (1u << (end - base)) : 0u);
          const int row = (__popc(before) + __popc(ends & ((2u << lane) - 1u))) & 31;
          const int rb = __shfl_sync(0xffffffffu, beg, row), rs = __shfl_sync(0xffffffffu, rstart, row);
          v[q] = f < total ? __ldg(p.csr_idx1 + (size_t)rs + (f - rb)) : make_int4(col, 0, 0, 0);
        }
        b0 += 32 * U_STEPS;
        if (b0 >= total) {
          k0 += U_WARPS * 32;
          live = k0 < ce;
          if (live) {
            const int2 seg = seg_next;
            seg_next = desc(k0 + U_WARPS * 32);
            open(seg);
          }
        }
      };
      const auto count = [&](const int4 (&v)[U_STEPS]) {
#pragma unroll
        for (int q = 0; q < U_STEPS; ++q) {
          unsigned t = (unsigned)(v[q].x - col - 1);
          k1d_up_count(acc_s, lane, t, t < sz);
#pragma unroll
          for (int e = 0; e < K1D_GAPS; ++e) {
            const unsigned g = (unsigned)k1d_gap(v[q], e);
            t += g;
            k1d_up_count(acc_s, lane, t, g != 0u && t < sz);
          }
        }
      };
      int4 va[U_STEPS], vb[U_STEPS];
      bool have_a = live;
      if (live) issue(va);
      while (have_a) {
        const bool have_b = live;
        if (live) issue(vb);
        count(va);
        if (!have_b) break;
        have_a = live;
        if (live) issue(va);
        count(vb);
      }
    }
    int4 wi_next = make_int4(0, 0, 0, 0);
    if (tid == 0) {
      it_next = failed ? p.n_range : it_next;
      if (it_next < p.n_range) wi_next = __ldg(p.worklist_up + it_next);
    }
    __syncthreads();
    PROF_MARK(8);

    // ---------------- sweep of the window's words: checksum, count >= 3 cells into the stage (past it: the loose list), clear;
    // every cell counts into deg[j] (fire-and-forget)
    {
      int ns = 0;
      uint4* acc4 = reinterpret_cast<uint4*>(acc);
      for (int i4 = tid; i4 < ((((size_c + 7) >> 3) + 3) >> 2); i4 += U_THREADS) {
        const uint4 w4 = acc4[i4];
        if (!(w4.x | w4.y | w4.z | w4.w)) continue;
        acc4[i4] = make_uint4(0u, 0u, 0u, 0u);
        const unsigned ww[4] = {w4.x, w4.y, w4.z, w4.w};
        unsigned bytes = 0u, any = 0u, m[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          bytes += (ww[e] & 0x0F0F0F0Fu) + ((ww[e] >> 4) & 0x0F0F0F0Fu);
          m[e] = nib_ge3(ww[e]);
          any |= m[e];
        }
        ns += (int)__dp4a(bytes, 0x01010101u, 0u);
        if (any) {
          const int c3 = __popc(m[0]) + __popc(m[1]) + __popc(m[2]) + __popc(m[3]);
          int pos = atomicAdd(&us.ncand, c3);
          // the staged cells form a prefix [0, nst) of the positions; a vector past the stage reserves its own slots
          const bool staged = pos + c3 <= U_STAGE;
          unsigned long long g = 0ull;
          if (staged) atomicAdd(&us.nst, c3);
          else g = atomicAdd(p.n_loose, (unsigned long long)c3);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            unsigned mm = m[e];
            while (mm) {
              const int q = (__ffs(mm) - 1) >> 2;
              mm &= mm - 1;
              int j = col + 1 + (i4 * 4 + e) * 8 + q;
              if (j >= n) j -= n;
              const unsigned cd = ((unsigned)j << 4) | ((ww[e] >> (q << 2)) & 15u);
              if (staged) {
                stage[pos++] = cd;
              } else {
                atomicAdd(p.deg + j, 1);
                if (g < (unsigned long long)p.loose_cap) p.loose[g] = ((u64)col << 32) | cd;
                else atomicExch(p.pair_fail, 1);
                ++g;
              }
            }
          }
        }
      }
      ns = __reduce_add_sync(0xffffffffu, ns);
      if (lane == 0 && ns) atomicAdd(&us.nibsum, ns);
    }
    if (tid == 0) { us.item = it_next; us.wi = wi_next; }  // every thread read this column's before the barrier above
    __syncthreads();
    const int nst = us.nst;
    if (tid == 0) {
      if (us.nibsum != adds) atomicExch(p.pair_fail, 1);  // a counter overflowed: the call falls back
      us.base = nst ? atomicAdd(p.n_own, (unsigned long long)nst) : 0ull;
      if (us.base + nst > (unsigned long long)p.pair_cap) atomicExch(p.pair_fail, 1);
      p.own_off[col] = (int)us.base;  // < pair_cap < 2^30 unless the call has fallen back
      p.own_n[col] = nst | (us.ncand > nst ? OWN_SPILLED : 0);
    }
    __syncthreads();
    const unsigned long long base = us.base;
    if (base + nst <= (unsigned long long)p.pair_cap)
      for (int t = tid; t < nst; t += U_THREADS) {
        const unsigned cd = stage[t];
        p.own[base + t] = cd;
        atomicAdd(p.deg + (cd >> 4), 1);
      }
    // every thread read nst before the barrier above; the next column's sweep counts after its first barrier
    if (tid == 0) { us.nibsum = 0; us.ncand = 0; us.nst = 0; }
    PROF_MARK(9);
  }
}

// Exchange (after the exclusive scan of deg into mir_off): every cell (i, j, count) of the own lists and of the loose list
// goes into the mirror list of j as (i << 4 | count), as a transpose by destination tile in two kernels whose writes stay
// local.  Tile t is the columns [t << tile_log2, (t + 1) << tile_log2), so the tile of a cell is j >> tile_log2 (no
// lookup), and its mirror region is [mir_off[c0], mir_off[c1]): columns are never split.
//   bucket: per CTA, a batch of X_BATCH source columns and a share of the loose list: a shared histogram over the
//           destination tiles, ONE returning global atomicAdd per (CTA, tile) on the tile's fill counter to reserve a run,
//           the cells grouped by tile in shared memory, then stored as runs of (j - c0 << 32 | i << 4 | count) into
//           `bucket`, which has the same offsets as mir: tile t's cells fill exactly its mirror region.  A run's stores
//           are issued together, so its sectors are complete in L2 before they are evicted (stored cell by cell as the
//           batch is read, they were not: the kernel took 1.3-2.3 ms at C5).  A batch larger than the stage is
//           stored cell by cell;
//   place:  one CTA per tile ranks its cells per destination column with shared-memory counters (started at the
//           columns' offsets in the region) and writes them into a shared copy of the region, which it then stores to mir
//           with coalesced full-sector writes (a region longer than X_STAGE is written to mir directly).  It zeroes deg
//           (spent: zero for the next call, also after a fallback, where nothing else runs) and tile_fill.
constexpr int X_THREADS = 512;     // threads of the bucket and place kernels
#ifndef B200_X_BATCH
#define B200_X_BATCH 32
#endif
constexpr int X_BATCH = B200_X_BATCH;  // source columns per bucket CTA (C5: ~6.9 K cells over 3 125 tiles; -D for A/B builds)
constexpr int X_ILP = 4;           // cells per lane in flight
constexpr int X_TILE_LOG2 = 6;     // default tile: 64 columns (C5: ~14 K cells, a 55 KB region)
constexpr int X_MAX_TILES = 12288; // the bucket kernel's per-tile arrays' bound (2 x 48 KB): wider tiles on larger catalogues
constexpr int X_BSTAGE = 10240;    // cells of a batch the bucket kernel groups in shared memory (80 KB: two CTAs per SM at C5)
constexpr int X_STAGE = 24576;     // region cells the place kernel stages in shared memory (96 KB: two CTAs per SM)

// Hands every cell of the bucket CTA's batch to fn(source column i, cell (j << 4 | count)): a warp per source column with
// X_ILP own-list loads in flight per lane, then the CTA's share of the loose list.
template <class Fn>
__device__ __forceinline__ void k1d_batch_cells(const KParams& p, Fn fn) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c1 = min(p.n_cols, (int)(blockIdx.x + 1) * X_BATCH);
  for (int i = blockIdx.x * X_BATCH + warp; i < c1; i += X_THREADS / 32) {
    const int so = p.own_off[i], n = p.own_n[i] & ~OWN_SPILLED;
    for (int t0 = 0; t0 < n; t0 += 32 * X_ILP) {
      unsigned cd[X_ILP];
#pragma unroll
      for (int q = 0; q < X_ILP; ++q) {
        const int t = t0 + 32 * q + lane;
        cd[q] = t < n ? p.own[so + t] : 0u;
      }
#pragma unroll
      for (int q = 0; q < X_ILP; ++q)
        if (t0 + 32 * q + lane < n) fn(i, cd[q]);
    }
  }
  const long long nl = (long long)min(*p.n_loose, (u64)p.loose_cap), G = gridDim.x;
  for (long long q = nl * blockIdx.x / G + threadIdx.x; q < nl * (blockIdx.x + 1) / G; q += X_THREADS) {
    const u64 c = p.loose[q];
    fn((int)(c >> 32), (unsigned)c);
  }
}

__global__ void __launch_bounds__(X_THREADS, 2) k1d_pair_bucket_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int n_batch;
  u64* stage = reinterpret_cast<u64*>(smem_raw);  // the batch's cells (j << 32 | i << 4 | count), grouped by tile
  const int L = p.tile_log2, n_tiles = ((p.n_cols - 1) >> L) + 1;
  // per destination tile: cells, then (run start in the bucket) - (start of the tile's group in the stage)
  int* hist = reinterpret_cast<int*>(stage + X_BSTAGE);
  int* next = hist + n_tiles;  // per destination tile: the next slot of its group
  if (*p.pair_fail) return;
  for (int t = threadIdx.x; t < n_tiles; t += X_THREADS) hist[t] = 0;
  if (threadIdx.x == 0) n_batch = 0;
  __syncthreads();
  k1d_batch_cells(p, [&](int, unsigned cd) { atomicAdd(&hist[cd >> (4 + L)], 1); });
  __syncthreads();
  for (int t = threadIdx.x; t < n_tiles; t += X_THREADS) {
    const int c = hist[t];
    if (!c) continue;
    const int g = p.mir_off[t << L] + atomicAdd(p.tile_fill + t, c), s = atomicAdd(&n_batch, c);
    hist[t] = g - s;
    next[t] = s;
    if (p.prof) { atomicAdd(p.prof + 12, 1ull); atomicAdd(p.prof + 13, (unsigned long long)c); }  // runs and cells
  }
  __syncthreads();
  const bool staged = n_batch <= X_BSTAGE;
  const unsigned mask = (1u << L) - 1u;
  k1d_batch_cells(p, [&](int i, unsigned cd) {
    const unsigned j = cd >> 4, lo = ((unsigned)i << 4) | (cd & 15u);
    const int r = atomicAdd(&next[j >> L], 1);
    if (staged) stage[r] = ((u64)j << 32) | lo;
    else p.bucket[hist[j >> L] + r] = ((u64)(j & mask) << 32) | lo;
  });
  if (!staged) return;
  __syncthreads();
  for (int k = threadIdx.x; k < n_batch; k += X_THREADS) {
    const u64 e = stage[k];
    const unsigned j = (unsigned)(e >> 32);
    p.bucket[hist[j >> L] + k] = ((u64)(j & mask) << 32) | (unsigned)e;
  }
}

// Persistent: CTA b places tiles b, b + gridDim.x, ...
__global__ void __launch_bounds__(X_THREADS, 2) k1d_pair_place_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int L = p.tile_log2;
  int* rank = reinterpret_cast<int*>(smem_raw);                      // per column of the tile: its next region position
  unsigned* stage = reinterpret_cast<unsigned*>(rank + (1 << L));    // the region
  const bool failed = *p.pair_fail;
  const int n_tiles = ((p.n_cols - 1) >> L) + 1;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int c0 = t << L, nc = min(1 << L, p.n_cols - c0);
    for (int k = threadIdx.x; k < nc; k += X_THREADS) p.deg[c0 + k] = 0;
    if (failed) continue;
    const int base = p.mir_off[c0], size = p.mir_off[c0 + nc] - base;
    if (size == 0) continue;
    for (int k = threadIdx.x; k < nc; k += X_THREADS) rank[k] = p.mir_off[c0 + k] - base;
    if (threadIdx.x == 0) p.tile_fill[t] = 0;  // its cells are exactly the region's: size of them
    __syncthreads();
    const bool staged = size <= X_STAGE;
    const u64* cells = p.bucket + base;
    for (int k0 = 0; k0 < size; k0 += X_THREADS * X_ILP) {
      u64 e[X_ILP];
#pragma unroll
      for (int q = 0; q < X_ILP; ++q) {
        const int k = k0 + q * X_THREADS + threadIdx.x;
        e[q] = k < size ? cells[k] : 0ull;
      }
#pragma unroll
      for (int q = 0; q < X_ILP; ++q)
        if (k0 + q * X_THREADS + threadIdx.x < size) {
          const int r = atomicAdd(&rank[(int)(e[q] >> 32)], 1);
          if (staged) stage[r] = (unsigned)e[q]; else p.mir[base + r] = (unsigned)e[q];
        }
    }
    __syncthreads();
    if (staged) {
      for (int k = threadIdx.x; k < size; k += X_THREADS) p.mir[base + k] = stage[k];
      __syncthreads();  // the region is stored before the next tile overwrites it
    }
  }
}

constexpr int S_WARPS = 4;            // columns (warps) per CTA of the select kernel
constexpr int S_CTAS = 6;             // CTAs per SM its registers are bounded for (shared memory allows that at C5)
constexpr int S_CAP = 4 * D_THREADS;  // the longest candidate list the select kernel decides (the K1-D kernel's key buffer)
constexpr int S_ILP = 12;             // candidates per lane in flight while the keys are built (C5: ~430 per column)
// shared memory of one select warp: its radix histogram, then the keys of a list of up to sel_cap candidates (the handle's
// bound, <= S_CAP: sized from the expected list lengths at create time, so that more warps fit on an SM), rounded to 16
// bytes so that every warp's histogram stays 16-byte aligned (select.cuh reads it as int4)
__host__ __device__ __forceinline__ int k1d_select_warp_bytes(int sel_cap) { return 256 * 4 + (sel_cap * 8 + 15) / 16 * 16; }

// One warp per column of the work list: keys from the column's own and mirror lists, the decision rule of sim_k1d_kernel's
// collected path, the K best, emit -- or the column goes to the redo list (all columns when the call has fallen back).
// No block barriers: a column's three dependent loads (list bounds, list, norm terms) overlap with the other warps' work.
template <int F>
__global__ void __launch_bounds__(32 * S_WARPS, S_CTAS) sim_k1d_select_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned char* mine = smem_raw + (size_t)(threadIdx.x >> 5) * k1d_select_warp_bytes(p.sel_cap);
  int* hist = reinterpret_cast<int*>(mine);
  u64* keys = reinterpret_cast<u64*>(mine + 256 * 4);
  const int lane = threadIdx.x & 31;
  const int item = blockIdx.x * S_WARPS + (threadIdx.x >> 5);
  if (item >= p.n_range) return;
  const int4 wi = __ldg(p.worklist + item);
  if (*(volatile int*)p.pair_fail) {
    if (lane == 0) { p.wl_redo[item] = wi; atomicAdd(p.n_redo, 1); }  // every column, in the work list's order
    return;
  }
  long long prof_t = p.prof ? clock64() : 0;
  const int col = wi.x, lc = wi.y, K = p.K;
  const int so = p.own_off[col], no = p.own_n[col];  // no < 0: OWN_SPILLED
  const int sm = p.mir_off[col], n = no + (p.mir_off[col + 1] - sm);
  bool ok = no >= 0 && n <= p.sel_cap;
  int n_have = 0;
  if (ok) {
    const float Ai = p.A[col];
    const unsigned* own = p.own + so;
    const unsigned* mir = p.mir + sm - no;  // candidate t >= no is mir[t]
    for (int t0 = 0; t0 < n; t0 += 32 * S_ILP) {
      unsigned cd[S_ILP];
      int2 bn[S_ILP];
#pragma unroll
      for (int q = 0; q < S_ILP; ++q) {
        const int t = t0 + 32 * q + lane;
        cd[q] = t < n ? (t < no ? own : mir)[t] : 0u;  // one load per candidate
      }
#pragma unroll
      for (int q = 0; q < S_ILP; ++q)
        if (t0 + 32 * q + lane < n) bn[q] = __ldg(p.BN + (cd[q] >> 4));
#pragma unroll
      for (int q = 0; q < S_ILP; ++q) {
        u64 key = 0ull;
        if (t0 + 32 * q + lane < n) {
          const float sv = sim_value<F>(p, (float)(cd[q] & 15u), Ai, __int_as_float(bn[q].x));
          if (sv > 0.f) key = (((u64)__float_as_uint(sv)) << 32) | (u64)(0xFFFFFFFFu - (unsigned)bn[q].y);
        }
        const unsigned b = __ballot_sync(0xffffffffu, key != 0ull);
        if (key) keys[n_have + __popc(b & ((1u << lane) - 1u))] = key;
        n_have += __popc(b);
      }
    }
    ok = false;
    if (n_have >= K) {
      // floor of the K-th best: (count 3, largest norm term); no count-2 / count-1 cell may reach it.  A count-c cell's
      // neighbour has at least c users, so its norm term is at least lvl_b<c> (an empty column's 0 does not count)
      const float fl = sim_value<F>(p, 3.f, Ai, p.tbnd[p.ntile]) * (1.f - 1e-6f);
      if (fl > 0.f) ok = !(sim_value<F>(p, 2.f, Ai, p.lvl_b2) >= fl) && !(sim_value<F>(p, 1.f, Ai, p.lvl_b1) >= fl);
    }
  }
  PROF_MARK_WARP(10);
  if (!ok) {
    if (lane == 0) p.wl_redo[atomicAdd(p.n_redo, 1)] = wi;
    return;
  }
  __syncwarp();
  const auto sel_key = [&](int q, u64& key) {
    key = keys[q];
    return true;
  };
  // the K-th largest key, so that exactly the K largest keys are >= it (0 when n_have == K: nothing is cut)
  const u64 thr = n_have > K ? radix_select<u64, 8, true>(WarpSelect{hist}, n_have, K, sel_key).thr : 0ull;
  // emit while compacting: the kept keys of every 32 take the next output slots in lane order
  const size_t out_base = (size_t)lc * K;
  int kept = 0;
  for (int t0 = 0; t0 < n_have; t0 += 32) {
    const int t = t0 + lane;
    const u64 k64 = t < n_have ? keys[t] : 0ull;
    const bool keep = t < n_have && k64 >= thr;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    if (keep)
      emit_entry(p, out_base + kept + __popc(b & ((1u << lane) - 1u)), (int)(0xFFFFFFFFu - (unsigned)k64),
                 __uint_as_float((unsigned)(k64 >> 32)));
    kept += __popc(b);
  }
  for (int t = kept + lane; t < K; t += 32) emit_entry(p, out_base + t, -1, 0.f);
  if (lane == 0) emit_count(p, lc, kept);
  PROF_MARK_WARP(11);
}

// tb[t] = norm term at neighbour min(t << D_TILE_LOG2, n_cols - 1), t = 0 .. ntile
__global__ void k1d_tile_bounds_kernel(const int2* __restrict__ BN, int n_cols, int ntile, float* tb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > ntile) return;
  tb[t] = __int_as_float(BN[min(t << D_TILE_LOG2, n_cols - 1)].x);
}

// entry m of a row written `copies` times (k1d layout above): row[m], then row[m - len] + n_cols
__device__ __forceinline__ int k1d_row_entry(const int* __restrict__ row, int len, int n_cols, int m) {
  return m < len ? row[m] : row[m - len] + n_cols;
}

// Walks one row in layout order and hands every chunk to emit(chunk number, chunk); returns the number of chunks.
template <class Emit>
__device__ __forceinline__ int k1d_row_chunks(const int* __restrict__ row, int len, int copies, int n_cols, Emit emit) {
  const int total = copies * len;
  int nch = 0;
  for (int m = 0; m < total; ++nch) {
    const int base = k1d_row_entry(row, len, n_cols, m++);
    unsigned long long g14 = 0ull;  // gaps 1..4, then 5..6
    unsigned g56 = 0u;
    for (int e = 0, prev = base; e < K1D_GAPS && m < total; ++e, ++m) {
      const int j = k1d_row_entry(row, len, n_cols, m);
      if (j - prev >= 65536) break;
      if (e < 4) g14 |= (unsigned long long)(j - prev) << (16 * e); else g56 |= (unsigned)(j - prev) << (16 * (e - 4));
      prev = j;
    }
    emit(nch, make_int4(base, (int)(unsigned)g14, (int)(unsigned)(g14 >> 32), (int)g56));
  }
  return nch;
}

// nchunk[u] = chunks of row u (one thread per row); rows from its exclusive scan poff.  In the fill, eight lanes per row
// walk it together (their loads are one broadcast) and lane l stores chunks l, l + 8, ...
__global__ void k1d_row_len_kernel(const int* __restrict__ csr_ptr, const int* __restrict__ csr_idx, int n_rows, int copies, int n_cols,
                                   int* nchunk) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n_rows) return;
  nchunk[u] = k1d_row_chunks(csr_idx + csr_ptr[u], csr_ptr[u + 1] - csr_ptr[u], copies, n_cols, [](int, int4) {});
}

__global__ void k1d_row_fill_kernel(const int* __restrict__ csr_ptr, const int* __restrict__ csr_idx, const int* __restrict__ poff,
                                    int n_rows, int copies, int n_cols, int4* rows) {
  const int u = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 3), l = threadIdx.x & 7;
  if (u >= n_rows) return;
  int4* out = rows + poff[u];
  k1d_row_chunks(csr_idx + csr_ptr[u], csr_ptr[u + 1] - csr_ptr[u], copies, n_cols, [=](int ch, int4 c) { if ((ch & 7) == l) out[ch] = c; });
}

// the chunk of a row (nch chunks) that holds entry m, whose value is v: the last one whose base is <= v.  The chunks before
// it hold at most seven entries each, so it is chunk m / 7 or a later one, and m / 7 itself unless a gap before entry m
// closed a chunk early: one look at the next base settles the usual case.
__device__ __forceinline__ int k1d_chunk_of(const int4* __restrict__ row, int nch, int m, int v) {
  int lo = m / (K1D_GAPS + 1), hi = nch;
  if (lo + 1 == nch || row[lo + 1].x > v) return lo;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (row[mid].x <= v) lo = mid; else hi = mid;
  }
  return lo;
}

// Per CSC entry q (user u, column c; csc_pos[q] = its position in the CSR, so its place in u's row is k = csc_pos[q] - r0):
// csc_seg[q] = the chunks that hold the first copy of u's row, for the K1-D kernel: x = first chunk, y = chunks; and
// col_adds[c] = the increments column c's rows produce there (entries - 1 per row).  With a doubled layout (win != nullptr)
// also win[q] = the chunks that hold the entry's window for the upper pass, entries k + 1 .. (last one <= c + size_c) of
// the doubled row, and win_work[c] = the increments of all of column c's windows (the upper pass's checksum target and
// the sort key of its longest-first order, with iota[c] = c as the value).  Increments are counted in the CSR, never from
// chunk counts.  One warp per column.
__global__ void k1d_csc_rows_kernel(const int* __restrict__ csc_ptr, const int* __restrict__ csc_idx, const int* __restrict__ csr_ptr,
                                    const int* __restrict__ csr_idx, const int* __restrict__ csc_pos, const int* __restrict__ poff,
                                    const int4* __restrict__ rows, int n_cols, int2* seg, int* col_adds, int2* win,
                                    unsigned long long* win_work, int* iota) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= n_cols) return;
  const int bound = c + k1d_window_size(n_cols, c);
  unsigned long long w = 0;
  int full = 0;
  for (int q = csc_ptr[c] + lane; q < csc_ptr[c + 1]; q += 32) {
    const int u = csc_idx[q];
    const int r0 = csr_ptr[u], len = csr_ptr[u + 1] - r0, s = poff[u], nch = poff[u + 1] - s;
    const int* row = csr_idx + r0;
    seg[q] = make_int2(s, k1d_chunk_of(rows + s, nch, len - 1, row[len - 1]) + 1);
    full += len - 1;
    if (!win) continue;
    // the window ends before the first entry in (k, k + len) whose index exceeds c + size_c (entry k + len is c + n)
    const int k = csc_pos[q] - r0;
    int lo = k + 1, hi = k + len;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (k1d_row_entry(row, len, n_cols, mid) <= bound) lo = mid + 1; else hi = mid;
    }
    int2 d = make_int2(0, 0);
    if (lo > k + 1) {
      const int first = k1d_chunk_of(rows + s, nch, k + 1, k1d_row_entry(row, len, n_cols, k + 1));
      d = make_int2(s + first, k1d_chunk_of(rows + s, nch, lo - 1, k1d_row_entry(row, len, n_cols, lo - 1)) - first + 1);
    }
    win[q] = d;
    w += (unsigned long long)(lo - k - 1);
  }
  full = __reduce_add_sync(0xffffffffu, full);
  if (lane == 0) col_adds[c] = full;
  if (!win) return;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
  if (lane == 0) { win_work[c] = w; iota[c] = c; }
}

// the upper pass's work list: every column (new numbering, in the order `perm`, work[k] = its window increments) as
// (new column, increments, csc range).  The increments are compared with a 32-bit nibble sum: their low 32 bits do.
__global__ void k1d_upper_worklist_kernel(const int* __restrict__ perm, const unsigned long long* __restrict__ work,
                                          const int* __restrict__ csc_ptr, int n_cols, int4* wl) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_cols) return;
  const int c = perm[k];
  wl[k] = make_int4(c, (int)(unsigned)work[k], csc_ptr[c], csc_ptr[c + 1]);
}

// ------------------------------------------------------------------------------------------------------
// Host side: a handle's K1-D and pair-path state, its set-up at create time (k1d_build) and its launches (k1d_launch).
// They take the similarity handle, b200_sim_s in sim_topk.cu, which holds a K1DState and is defined after this header:
// hence the template parameter.  What the kernels read lives in the handle's KParams `base`; this is the rest.
// ------------------------------------------------------------------------------------------------------
struct K1DState {
  // routing: on by default for binary data with >= k1c_min_cols columns; whether the handle qualified; the expected hits per
  // neighbour (gathered entries / n_cols) below which a column takes K1-D; the last launch's split of the columns
  bool want_k1c = true, k1c = false;
  double k1c_lambda = 0.75;
  int k1c_min_cols = 32768;
  int n_sparse_last = 0, n_dense_last = 0;
  sim_kernel_t kernel = nullptr, select_kernel = nullptr;  // the instances of the handle's formula
  // second row layout with one window, CSC-side row locations, norm tile bounds, redo count, work list, CTAs per SM and
  // dynamic shared memory of the K1-D kernel; the new index and CSC range of every column, for the host's work lists
  DevBuf<int4> csr_idx1, worklist;
  DevBuf<int> col_adds, fail;
  DevBuf<int2> csc_seg;
  DevBuf<float> tbnd;
  int ctas_per_sm = 0;
  size_t smem1_bytes = 0;
  std::vector<int> h_old2new, h_csc_ptr;
  // pair path: row windows, the upper pass's work list (every column), own lists (capacity from the expected pair count)
  // with their per-column start and length, loose list, mirror lists (deg: per-column counts, zero between calls), the
  // exchange's bucket buffer and destination tiles (fill counters: zero between calls; the columns per tile requested,
  // normally 2^X_TILE_LOG2), control words (own and loose fill, fallback flag, redo count), redo list, scan scratch (all
  // allocated by the first call that takes the path: k1d_pair_buffers), upper-pass and select geometry
  DevBuf<int2> csc_win;
  DevBuf<int4> worklist_up, wl_redo;
  DevBuf<unsigned> own, mir;
  DevBuf<u64> loose, bucket;
  double pairs_expected = 0.0;
  DevBuf<int> own_off, own_n, deg, mir_off, pair_ctl, tile_fill;
  int tile_log2_req = X_TILE_LOG2;
  DevBuf<unsigned char> scan_tmp;
  size_t scan_tmp_bytes = 0, smem_up_bytes = 0, smem_sel_bytes = 0;
  int ctas_up = 0;
  bool pair_path_last = false;  // the cached routing qualifies for the pair path
};

// Whether the K1-D pair path pays on this data.  It saves about half of a K1-D pass when the select kernel decides a column
// itself, and costs a full K1-D pass more for every column it hands back, so it is taken only when at least 90 % of the
// non-empty columns are expected to pass the select kernel's rule: with users drawn independently, column c has
// n_cols * P(Poisson(lambda_c) >= 3) cells with count >= 3 (lambda_c = gathered entries off the diagonal / n_cols), which
// must reach K, and
// no count-2 / count-1 cell may reach the floor sim(3, largest norm term).  Sets the smallest norm terms of the neighbours
// a count-1 / count-2 cell can have, the expected number of pairs (which sizes the pair list), and the longest list the
// select kernel decides: the largest expected list plus six standard deviations (Poisson) and 32, in multiples of 8, at
// most S_CAP.  A longer list is redone exactly; the bound only sizes the select kernel's shared memory, so that more of
// its warps fit on an SM (C5: expected lists of 243 to 778, sel_cap 984, six CTAs per SM instead of three).
template <class Handle>
bool k1d_pair_gate(Handle* h, const int* d_cnt, cudaStream_t st) {
  KParams& p = h->base;
  const int n = p.n_cols;
  std::vector<int> cnt((size_t)n);
  std::vector<int2> bn((size_t)n);
  std::vector<float> a((size_t)n);
  B200_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(bn.data(), h->BN.get(), sizeof(int2) * (size_t)n, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(a.data(), h->A.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  auto bval = [&](int j) { float b; std::memcpy(&b, &bn[(size_t)j].x, sizeof b); return b; };
  float b1 = FLT_MAX, b2 = FLT_MAX;
  for (int j = 0; j < n; ++j) {
    if (cnt[(size_t)j] >= 1) b1 = std::min(b1, bval(j));
    if (cnt[(size_t)j] >= 2) b2 = std::min(b2, bval(j));
  }
  p.lvl_b1 = b1;
  p.lvl_b2 = b2;
  const float bmax = bval(n - 1);
  long long nonempty = 0, pass = 0;
  double cells = 0.0, est_max = 0.0;
  with_formula<F_PROD, F_NONORM, F_JACCARD, F_DICE, F_TVERSKY>(h->formula, [&](auto f) {
    constexpr int F = decltype(f)::value;
    for (int c = 0; c < n; ++c) {
      if (cnt[(size_t)c] == 0) continue;
      ++nonempty;
      const double lam = (double)(h->h_work[(size_t)bn[(size_t)c].y] - (unsigned long long)cnt[(size_t)c]) / (double)n;
      const double est = (double)n * std::max(0.0, 1.0 - std::exp(-lam) * (1.0 + lam + 0.5 * lam * lam));
      cells += est;
      est_max = std::max(est_max, est);
      const float ai = a[(size_t)c];
      const float fl = sim_value<F>(p, 3.f, ai, bmax) * (1.f - 1e-6f);
      if (est >= (double)p.K && fl > 0.f && !(sim_value<F>(p, 2.f, ai, b2) >= fl) && !(sim_value<F>(p, 1.f, ai, b1) >= fl)) ++pass;
    }
  });
  h->k1d.pairs_expected = 0.5 * cells;
  p.sel_cap = (int)std::min<double>(std::ceil((est_max + 6.0 * std::sqrt(est_max) + 32.0) / 8.0) * 8.0, (double)S_CAP);
  return nonempty > 0 && (double)pass >= 0.9 * (double)nonempty;
}

// K1-D's part of the handle's set-up, for binary data whose formula K1-D serves: the row layout and its CSC-side locations,
// the CTAs per SM that fit, the pair path's gate and its upper pass's work list.  Points h->base at the buffers it keeps.
// d_cnt: users per column; d_csc_pos: the CSR position of every CSC entry; h->csr_idx is still the unpadded CSR.
template <class Handle>
void k1d_build(Handle* h, const int* d_cnt, const int* d_csc_pos, cudaStream_t st) {
  K1DState& k = h->k1d;
  KParams& b = h->base;
  const int n_rows = h->n_rows, n_cols = b.n_cols;
  const long long nnz = h->nnz;
  with_formula<F_PROD, F_NONORM, F_JACCARD, F_DICE, F_TVERSKY>(h->formula, [&](auto f) {
    k.kernel = sim_k1d_kernel<decltype(f)::value>;
    k.select_kernel = sim_k1d_select_kernel<decltype(f)::value>;
  });
  const bool f_ok_c = h->formula == F_PROD || h->formula == F_NONORM || h->formula == F_JACCARD || h->formula == F_DICE ||
                      (h->formula == F_TVERSKY && b.ta >= 0.f && b.tb >= 0.f);  // decreasing in the neighbour's norm term
  if (!h->binary || !k.want_k1c || !f_ok_c || nnz == 0 || n_cols < k.k1c_min_cols) return;
  DevBuf<unsigned long long> win_work;  // upper-pass work per new column, and the new column indices
  DevBuf<int> win_iota;
  {
    // every row twice, back to back, for the pair path's windows -- once when the doubled layout might not fit 32-bit chunk
    // positions: the K1-D kernel reads only the first copy, and the handle does not take the pair path.  A row never has
    // more chunks than entries, so the bound on the entries that the four-per-chunk layout needed still covers every matrix,
    // whatever its gaps
    const int copies = 2 * (long long)nnz + 3ll * n_rows < (1ll << 31) ? 2 : 1;
    DevBuf<int> len1((size_t)n_rows + 1), poff1((size_t)n_rows + 1);
    B200_CUDA(cudaMemsetAsync(len1.get() + n_rows, 0, sizeof(int), st));
    k1d_row_len_kernel<<<div_up(n_rows, 256), 256, 0, st>>>(h->csr_ptr.get(), h->csr_idx.get(), n_rows, copies, n_cols, len1.get());
    count_launch();
    size_t tb1 = 0;
    B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb1, len1.get(), poff1.get(), n_rows + 1, st));
    DevBuf<unsigned char> tmp1(tb1 + 16);
    B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp1.get(), tb1, len1.get(), poff1.get(), n_rows + 1, st)); count_launch();
    int total1 = 0;
    B200_CUDA(cudaMemcpyAsync(&total1, poff1.get() + n_rows, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    k.csr_idx1.alloc((size_t)total1 + 2);
    k1d_row_fill_kernel<<<div_up((long long)n_rows * 8, 256), 256, 0, st>>>(h->csr_ptr.get(), h->csr_idx.get(), poff1.get(), n_rows,
                                                                           copies, n_cols, k.csr_idx1.get()); count_launch();
    k.col_adds.alloc((size_t)n_cols);
    k.csc_seg.alloc((size_t)nnz + 2);
    B200_CUDA(cudaMemsetAsync(k.csc_seg.get() + nnz, 0, 2 * sizeof(int2), st));
    if (copies == 2) {
      k.csc_win.alloc((size_t)nnz);
      win_work.alloc((size_t)n_cols);
      win_iota.alloc((size_t)n_cols);
    }
    k1d_csc_rows_kernel<<<div_up((long long)n_cols * 32, 256), 256, 0, st>>>(h->csc_ptr.get(), h->csc_idx.get(), h->csr_ptr.get(),
                                                                             h->csr_idx.get(), d_csc_pos, poff1.get(),
                                                                             k.csr_idx1.get(), n_cols, k.csc_seg.get(),
                                                                             k.col_adds.get(), k.csc_win.get(), win_work.get(),
                                                                             win_iota.get()); count_launch();
    B200_CUDA(cudaStreamSynchronize(st));
  }
  // ---- geometry and eligibility
  const int win1 = ((n_cols + 7) / 8) * 8;
  b.ntile = (n_cols + (1 << D_TILE_LOG2) - 1) >> D_TILE_LOG2;
  b.bm_words = ((win1 / 8 + 1) + 3) / 4 * 4;
  const long long fixed = (long long)b.bm_words * 4 + ((long long)b.ntile + 1) * 4 + (long long)b.ntile * 4 + 32;
  // two CTAs per SM when both fit (each CTA also pays its static shared memory and the 1 KB the hardware reserves)
  cudaFuncAttributes fa{};
  B200_CUDA(cudaFuncGetAttributes(&fa, k.kernel));
  int dev = 0, sm_total = 0, max_smem = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sm_total, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
  B200_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const long long need_keys = (long long)b.K + (1ll << D_TILE_LOG2) + 128;  // a pruned buffer always takes one more tile
  for (int ctas = 2; ctas >= 1 && !k.k1c; --ctas) {
    long long avail = (long long)sm_total / ctas - (long long)fa.sharedSizeBytes - 1024;
    avail = std::min<long long>(avail, (long long)max_smem - (long long)fa.sharedSizeBytes);
    const long long keys = std::min<long long>((avail - fixed) / 8, 4 * D_THREADS);
    if (keys >= need_keys) {
      k.ctas_per_sm = ctas;
      b.cap_d = (int)keys;
      k.smem1_bytes = (size_t)(fixed + keys * 8);
      k.k1c = true;
    }
  }
  if (k.k1c) {
    k.tbnd.alloc((size_t)b.ntile + 1);
    k1d_tile_bounds_kernel<<<div_up(b.ntile + 1, 128), 128, 0, st>>>(h->BN.get(), n_cols, b.ntile, k.tbnd.get()); count_launch();
    k.fail.alloc(1);
    k.worklist.alloc((size_t)n_cols);
    k.h_old2new.resize((size_t)n_cols);
    k.h_csc_ptr.resize((size_t)n_cols + 1);
    B200_CUDA(cudaMemcpyAsync(k.h_old2new.data(), h->old2new.get(), sizeof(int) * (size_t)n_cols, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(k.h_csc_ptr.data(), h->csc_ptr.get(), sizeof(int) * ((size_t)n_cols + 1), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    raise_smem_limit(k.kernel, k.smem1_bytes);
    // the whole unified L1 / shared array as shared memory: without it the driver sizes the carve-out for ONE block and the
    // second CTA of an SM never becomes resident
    B200_CUDA(cudaFuncSetAttribute(k.kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));

    // pair path: needs the doubled row layout; the upper pass needs the half-window counters and the stage (up to U_CTAS
    // CTAs per SM as they fit), and it only pays when the select kernel can decide most columns itself (k1d_pair_gate); its
    // buffers are allocated by the first call that takes it
    cudaFuncAttributes fu{};
    B200_CUDA(cudaFuncGetAttributes(&fu, sim_k1d_upper_kernel));
    k.smem_up_bytes = ((size_t)k1d_upper_words(n_cols) + U_STAGE) * 4;
    k.ctas_up = 0;
    for (int ctas = U_CTAS; ctas >= 1 && k.ctas_up == 0 && k.csc_win.n > 0; --ctas)
      if ((long long)k.smem_up_bytes <= std::min<long long>((long long)sm_total / ctas - 1024, (long long)max_smem) - (long long)fu.sharedSizeBytes)
        k.ctas_up = ctas;
    if (k.ctas_up > 0 && !k1d_pair_gate(h, d_cnt, st)) k.ctas_up = 0;
    if (k.ctas_up > 0) {
      raise_smem_limit(sim_k1d_upper_kernel, k.smem_up_bytes);
      B200_CUDA(cudaFuncSetAttribute(sim_k1d_upper_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
      // the launch passes this handle's size; the limit is the same for every handle that shares the kernel
      k.smem_sel_bytes = (size_t)S_WARPS * k1d_select_warp_bytes(b.sel_cap);
      B200_CUDA(cudaFuncSetAttribute(k.select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S_WARPS * k1d_select_warp_bytes(S_CAP)));
      B200_CUDA(cudaFuncSetAttribute(k.select_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
      k.worklist_up.alloc((size_t)n_cols);
      // the upper pass's longest-first order: every column by descending window work (empty columns do nothing there)
      DevBuf<unsigned long long> keys_out((size_t)n_cols);
      DevBuf<int> perm((size_t)n_cols);
      size_t tb = 0;
      B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, tb, win_work.get(), keys_out.get(), win_iota.get(), perm.get(), n_cols, 0, 64, st));
      DevBuf<unsigned char> tmp(tb + 16);
      B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(tmp.get(), tb, win_work.get(), keys_out.get(), win_iota.get(), perm.get(), n_cols, 0, 64, st));
      k1d_upper_worklist_kernel<<<div_up(n_cols, 256), 256, 0, st>>>(perm.get(), keys_out.get(), h->csc_ptr.get(), n_cols, k.worklist_up.get());
      count_launch(5);
      B200_CUDA(cudaStreamSynchronize(st));
    }
  }
  if (!k.k1c) { k.csr_idx1.release(); k.csc_seg.release(); k.col_adds.release(); }
  if (k.ctas_up == 0) k.csc_win.release();
  b.tbnd = k.tbnd.get(); b.csr_idx1 = k.csr_idx1.get(); b.csc_seg = k.csc_seg.get(); b.col_adds = k.col_adds.get();
  b.worklist = k.worklist.get(); b.fail = k.fail.get();
  b.csc_win = k.csc_win.get(); b.worklist_up = k.worklist_up.get();
}

// The pair path's buffers, allocated by the first call that takes it, and its destination tiles, allocated again after
// b200_sim_debug_pair_lists changed their width.  Points h->base at them, before the call copies its parameters from there.
template <class Handle>
void k1d_pair_buffers(Handle* h, cudaStream_t st) {
  K1DState& k = h->k1d;
  KParams& b = h->base;
  const int n = b.n_cols;
  if (k.own.n == 0) {
    // the own lists hold twice the expected pairs (a fuller list sets the fallback flag), the loose list (cells past a
    // column's stage: rare) a quarter of that, the mirror lists and the exchange's bucket buffer both; positions stay below
    // 2^31
    b.pair_cap = std::min<long long>((long long)(2.0 * k.pairs_expected) + (1 << 16), (1ll << 30) - 1);
    b.loose_cap = b.pair_cap / 4 + (1 << 16);
    k.own.alloc((size_t)b.pair_cap);
    k.loose.alloc((size_t)b.loose_cap);
    k.mir.alloc((size_t)(b.pair_cap + b.loose_cap));
    k.bucket.alloc((size_t)(b.pair_cap + b.loose_cap));
    k.own_off.alloc((size_t)n);
    k.own_n.alloc((size_t)n);
    k.deg.alloc((size_t)n + 1);
    k.mir_off.alloc((size_t)n + 1);
    k.pair_ctl.alloc(6);  // [0..1] own fill (64-bit), [2] fallback flag, [3] redo count, [4..5] loose fill (64-bit)
    k.wl_redo.alloc((size_t)n);
    B200_CUDA(cudaMemsetAsync(k.deg.get(), 0, sizeof(int) * ((size_t)n + 1), st));
    B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, k.scan_tmp_bytes, k.deg.get(), k.mir_off.get(), n + 1, st));
    k.scan_tmp.alloc(k.scan_tmp_bytes + 16);
    b.own = k.own.get(); b.own_off = k.own_off.get(); b.own_n = k.own_n.get();
    b.n_own = reinterpret_cast<u64*>(k.pair_ctl.get());
    b.pair_fail = k.pair_ctl.get() + 2; b.n_redo = k.pair_ctl.get() + 3;
    b.loose = k.loose.get(); b.n_loose = reinterpret_cast<u64*>(k.pair_ctl.get() + 4);
    b.deg = k.deg.get(); b.mir_off = k.mir_off.get(); b.mir = k.mir.get(); b.wl_redo = k.wl_redo.get(); b.bucket = k.bucket.get();
  }
  if (k.tile_fill.n == 0) {
    // destination tiles of the exchange: the requested columns per tile, doubled while the bucket kernel's per-tile arrays
    // would not fit (C5: 3 125 tiles of 64 columns)
    b.tile_log2 = k.tile_log2_req;
    while (((n - 1) >> b.tile_log2) + 1 > X_MAX_TILES) ++b.tile_log2;
    const size_t nt = (size_t)((n - 1) >> b.tile_log2) + 1;
    k.tile_fill.alloc(nt);
    B200_CUDA(cudaMemsetAsync(k.tile_fill.get(), 0, sizeof(int) * nt, st));
    raise_smem_limit(k1d_pair_bucket_kernel, sizeof(u64) * X_BSTAGE + 2 * sizeof(int) * nt);
    raise_smem_limit(k1d_pair_place_kernel, sizeof(int) * (((size_t)1 << b.tile_log2) + X_STAGE));
    B200_CUDA(cudaFuncSetAttribute(k1d_pair_place_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    B200_CUDA(cudaFuncSetAttribute(k1d_pair_bucket_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    b.tile_fill = k.tile_fill.get();
  }
}

// K1-D's part of a launch: the n_sparse > 0 columns the routing sent to it, with the call's parameters p.  On the pair path
// the upper pass (own lists, deg) -> scan -> exchange (bucket, place: mirror lists) -> select, and the select kernel's redo
// list (every column after a fallback) goes through the K1-D kernel; otherwise the K1-D kernel takes the columns itself.
// Either way the columns with an overflowed counter are appended to the window kernel's list, whose length the window
// kernel then reads from the device (p.n_range_dev): no host round trip between the launches.
template <class Handle>
void k1d_launch(Handle* h, KParams& p, int n_sparse, bool pair_path, cudaStream_t st) {
  K1DState& k = h->k1d;
  const int n = p.n_cols, grid = std::min(n_sparse, h->n_sm * k.ctas_per_sm);
  B200_CUDA(cudaMemcpyAsync(p.fail, &k.n_dense_last, sizeof(int), cudaMemcpyHostToDevice, st));
  KParams q = p;
  q.n_range = n_sparse;
  if (pair_path) {
    B200_CUDA(cudaMemsetAsync(k.pair_ctl.get(), 0, 6 * sizeof(int), st));
    q.n_range = n;  // the upper pass's work list holds every column
    sim_k1d_upper_kernel<<<std::min(n, h->n_sm * k.ctas_up), U_THREADS, k.smem_up_bytes, st>>>(q);
    q.n_range = n_sparse;
    B200_CUDA(cudaGetLastError());
    size_t tb = k.scan_tmp_bytes;
    B200_CUDA(cub::DeviceScan::ExclusiveSum(k.scan_tmp.get(), tb, k.deg.get(), k.mir_off.get(), n + 1, st));
    k1d_pair_bucket_kernel<<<div_up(n, X_BATCH), X_THREADS, sizeof(u64) * X_BSTAGE + 2 * sizeof(int) * k.tile_fill.n, st>>>(q);
    k1d_pair_place_kernel<<<2 * h->n_sm, X_THREADS, sizeof(int) * (((size_t)1 << p.tile_log2) + X_STAGE), st>>>(q);
    B200_CUDA(cudaGetLastError());
    k.select_kernel<<<div_up(n_sparse, S_WARPS), 32 * S_WARPS, k.smem_sel_bytes, st>>>(q);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(int), st));
    q.worklist = k.wl_redo.get();
    q.n_range_dev = p.n_redo;
    k.kernel<<<grid, D_THREADS, k.smem1_bytes, st>>>(q);
    B200_CUDA(cudaGetLastError());
    count_launch(7);
  } else {
    k.kernel<<<grid, D_THREADS, k.smem1_bytes, st>>>(q);
    B200_CUDA(cudaGetLastError());
    count_launch();
  }
  B200_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(int), st));
  p.n_range_dev = p.fail;
}
