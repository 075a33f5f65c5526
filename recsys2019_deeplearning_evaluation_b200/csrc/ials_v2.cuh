// K4 on the tensor cores, second generation (sm_90a): implicit-ALS half epochs for n_factors <= 256.
//
// Replaces MatrixFactorization/IALSRecommender.py:137-201 like ials.cu (per warm row:  A = Y_p^T diag(c - 1) Y_p,
// B = Y^T Y + A + reg I,  x = B^-1 Y_p^T c), with the dense contraction on the tensor cores (wgmma) as BASELINE.json's
// north_star asks.
//
// Why a second generation.  ials.cu accumulates the Gram in fp64 registers and factors a packed fp64 matrix that no longer
// fits shared memory above 208 factors, so it is slow there.  The first tensor-core kernel (one 128 x 128 accumulator,
// fp64 Cholesky) only covered 128 factors and was slower than the fp64 kernel it was meant to replace -- scalar staging and an unblocked factorisation.  Here:
//   * Gram on the tensor core, 3xTF32 (fp32-accurate).  The profile's factor rows are scaled by sqrt(c - 1) while they are
//     staged, so ONE operand serves both sides of  A = (sqrt(c-1) Y_p)^T (sqrt(c-1) Y_p): per 32 profile entries a
//     256 x 32 hi tile and a lo tile (K-major wgmma layout, 128-bit shared stores, two stages).  Only the lower triangle is
//     formed, in register accumulators of the four warpgroups.  Above 128 factors (TWO) it is cut into the 20 blocks of
//     64 rows x 32 columns that meet the lower triangle of 256 x 256; block b (row-major order) belongs to warpgroup b % 4
//     (5 blocks, 80 fp32 per thread, three m64n32k8 wgmmas per block and 8 profile entries).  Up to 128 factors each
//     warpgroup owns one 64 x 64 block of the 128 x 128 matrix (the fourth one, above the diagonal, is discarded).  Every
//     warpgroup issues the same instruction sequence whatever n_factors is, so the wgmmas pipeline.  The staging of the
//     next step overlaps the wgmmas of this one.
//   * B in fp32, lower triangle, rows padded to 16 bytes (133 KB at 256 factors: it takes over the staging buffers), then a
//     right-looking blocked Cholesky with 32-wide panels: the diagonal block in the registers of one warp (shuffles), the
//     panel by one thread per row, the trailing update by warps that own 16 x 32 blocks of it so that their 128-bit
//     operand loads are broadcasts; the inverses of the diagonal blocks are kept for the solves.
//   * The solution is refined against the EXACT operator in fp64,  r = b - (Y^T Y x + Y_p^T((c-1) .* (Y_p x)) + reg x),
//     matrix-free, twice: only the fp32 factor is approximate, so each step contracts the error by ~cond * 1e-7.  A row whose
//     residual does not contract (ill-conditioned system) raises `redo`; the host then repeats the half epoch with ials.cu.
// Y^T Y comes from gram_kernel (ials.cu, fp64).  One CTA (512 threads) per SM, rows strided over the grid.
#pragma once
#include "gemm_tc.cuh"

namespace b200 {
namespace ials2 {

constexpr int T = 512;                   // 16 warps: the phases between the barriers are latency-bound, more warps hide more of it
constexpr int NW = T / 32;
constexpr int KC = 32;                   // profile entries per step
constexpr int STAGES = 2;
constexpr int TILE = 256 * KC * 4;       // one 256 x 32 fp32 tile: 32 KB
constexpr int NB = 32;                   // Cholesky panel width
constexpr int NBP = NB + 1;              // row stride of the stored diagonal-block inverses (no shared bank across rows)
constexpr int GB = 5;                    // Gram blocks (64 x 32) per warpgroup: 20 blocks of the lower triangle / 4

// block b of the lower triangle of a 256 x 256 matrix in 64 x 32 blocks, row-major: rows 64 rb.., columns 32 cb..
__device__ __forceinline__ void gram_block(int b, int& rb, int& cb) {
  rb = b < 2 ? 0 : b < 6 ? 1 : b < 12 ? 2 : 3;
  cb = b - (rb == 0 ? 0 : rb == 1 ? 2 : rb == 2 ? 6 : 12);
}

// lower triangle, row r starts at roff(r) floats: rows are padded to multiples of 4 floats so that every 4-aligned column
// offset of every row is 16-byte aligned
__device__ __host__ __forceinline__ int roff(int r) { const int q = r >> 2, m = r & 3; return 4 * (q + 1) * (2 * q + m); }

struct Smem {
  float* L;        // padded lower triangle (aliases the staging tiles)
  unsigned char* tiles;
  double *b0, *xs, *rs, *part;  // rhs, solution, residual / correction, [NW][f] partial sums
  float* dinv;     // [f / 32][32][33] inverses of the diagonal blocks of L (lower triangular, row-major, padded rows)
  float* sw;       // [KC] sqrt(c - 1) of the step's entries
  double* cw;      // [KC] c
  int* rk;         // [KC] factor-row indices (-1 past the profile)
  float* rdiag;    // [NB] reciprocals of the current diagonal block's diagonal
};

// ---- L z = v (forward) or L^T z = v (backward) in place on v (fp64), blocked by NB with the stored diagonal-block inverses
__device__ __forceinline__ void solve_forward(const Smem& S, double* v, int f) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int k0 = 0; k0 < f; k0 += NB) {
    const int nb = min(NB, f - k0);
    if (warp == 0) {  // z_blk = inv(L11) v_blk
      const float* inv = S.dinv + (k0 / NB) * NB * NBP;
      double z = 0.0;
      if (lane < nb)
        for (int c = 0; c <= lane; ++c) z += (double)inv[lane * NBP + c] * v[k0 + c];
      __syncwarp();
      if (lane < nb) v[k0 + lane] = z;
    }
    __syncthreads();
    const int r = k0 + nb + tid;  // rows below the block: v[r] -= L[r, blk] z_blk
    if (r < f) {
      const float* Lr = S.L + roff(r) + k0;
      double s = 0.0;
      for (int c = 0; c < nb; ++c) s += (double)Lr[c] * v[k0 + c];
      v[r] -= s;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ void solve_backward(const Smem& S, double* v, int f) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblk = (f + NB - 1) / NB;
  for (int kb = nblk - 1; kb >= 0; --kb) {
    const int k0 = kb * NB, nb = min(NB, f - k0);
    if (warp == 0) {  // x_blk = inv(L11)^T v_blk
      const float* inv = S.dinv + kb * NB * NBP;
      double z = 0.0;
      if (lane < nb)
        for (int c = lane; c < nb; ++c) z += (double)inv[c * NBP + lane] * v[k0 + c];
      __syncwarp();
      if (lane < nb) v[k0 + lane] = z;
    }
    __syncthreads();
    if (tid < k0) {  // columns left of the block: v[c] -= sum_r L[k0 + r, c] x[k0 + r]
      double s = 0.0;
      for (int r = 0; r < nb; ++r) s += (double)S.L[roff(k0 + r) + tid] * v[k0 + r];
      v[tid] -= s;
    }
    __syncthreads();
  }
}

template <bool TWO>
__global__ void __launch_bounds__(T, 1) ials_rows_v2_kernel(const int* __restrict__ rows, int n_solve, const int* __restrict__ ptr,
                                                            const int* __restrict__ idx, const float* __restrict__ conf,
                                                            const double* __restrict__ Y, const double* __restrict__ YtY, int f,
                                                            double reg, double* X, int* info, int* redo, int n_refine) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ double s_norm[3];  // |r|^2 before the last / the first correction, |b|^2
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  Smem S;
  {
    const size_t lbytes = (size_t)roff(f) * 4;
    size_t o = std::max<size_t>(lbytes, (size_t)STAGES * 2 * TILE);
    o = (o + 127) & ~(size_t)127;
    S.L = reinterpret_cast<float*>(smem);
    S.tiles = smem;
    S.b0 = reinterpret_cast<double*>(smem + o); o += sizeof(double) * f;
    S.xs = reinterpret_cast<double*>(smem + o); o += sizeof(double) * f;
    S.rs = reinterpret_cast<double*>(smem + o); o += sizeof(double) * f;
    S.part = reinterpret_cast<double*>(smem + o); o += sizeof(double) * NW * f;
    S.cw = reinterpret_cast<double*>(smem + o); o += sizeof(double) * KC;
    S.dinv = reinterpret_cast<float*>(smem + o); o += sizeof(float) * ((f + NB - 1) / NB) * NB * NBP;
    S.sw = reinterpret_cast<float*>(smem + o); o += sizeof(float) * KC;
    S.rk = reinterpret_cast<int*>(smem + o); o += sizeof(int) * KC;
    S.rdiag = reinterpret_cast<float*>(smem + o);
  }
  // this warpgroup's Gram blocks (64 rows x BW columns): their first row / column and the shared-memory byte offsets of their
  // A (64 tile rows) and B (BW tile rows) operands; one tile row group of 8 is 1024 B
  constexpr int NBLK = TWO ? GB : 1, BW = TWO ? 32 : 64;
  const int wg = tid >> 7, t = tid & 127;
  int r0[NBLK], c0[NBLK];
  uint32_t a_off[NBLK], b_off[NBLK];
#pragma unroll
  for (int j = 0; j < NBLK; ++j) {
    int rb, cb;
    if (TWO) gram_block(wg + 4 * j, rb, cb);
    else { rb = (wg == 1 || wg == 2) ? 1 : 0; cb = wg >> 1; }
    r0[j] = rb * 64;
    c0[j] = cb * BW;
    a_off[j] = (uint32_t)r0[j] * 128u;
    b_off[j] = (uint32_t)c0[j] * 128u;
  }
  float acc[NBLK][BW / 2];

  unsigned gk = 0;  // steps issued by this CTA so far (all rows): stage = gk & 1
  for (int srow = blockIdx.x; srow < n_solve; srow += gridDim.x) {
    const int row = rows[srow];
    const int p0 = ptr[row], p1 = ptr[row + 1];
    const int nk = (p1 - p0 + KC - 1) / KC;

    // ================= Gram on the tensor core
    double my_rhs = 0.0;  // threads m and m + 256 each hold half of b0[m] = (Y_p^T c)[m]  (IALSRecommender.py:201)
#pragma unroll
    for (int j = 0; j < NBLK; ++j)
#pragma unroll
      for (int i = 0; i < BW / 2; ++i) acc[j][i] = 0.f;
    for (int kb = 0; kb < nk; ++kb, ++gk) {
      const int s = (int)(gk & 1u);
      unsigned char* t_hi = S.tiles + (size_t)(s * 2 + 0) * TILE;
      unsigned char* t_lo = S.tiles + (size_t)(s * 2 + 1) * TILE;
      __syncthreads();  // rk / sw / cw of the previous step are consumed
      if (tid < KC) {
        const int q = p0 + kb * KC + tid;
        const float c = q < p1 ? conf[q] : 1.f;
        S.rk[tid] = q < p1 ? idx[q] : -1;
        S.sw[tid] = sqrtf(fmaxf(c - 1.f, 0.f));
        S.cw[tid] = q < p1 ? (double)c : 0.0;
      }
      __syncthreads();
      // tile(m, k) = sqrt(c_k - 1) * Y[rk[k]][m]; thread = (factor m, half of the step's entries), four entries per 128-bit
      // store; zero past f / the profile
      {
        const int m = tid & 255, kh = tid >> 8;
#pragma unroll
        for (int kq = kh * (KC / 8); kq < (kh + 1) * (KC / 8); ++kq) {
          float h[4], l[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int k = kq * 4 + e;
            const int r = S.rk[k];
            const double y = (r >= 0 && m < f) ? Y[(size_t)r * f + m] : 0.0;
            my_rhs += S.cw[k] * y;
            tc::split_tf32((float)y * S.sw[k], h[e], l[e]);
          }
          const uint32_t off = tc::tile_offset(m, kq * 4);
          *reinterpret_cast<float4*>(t_hi + off) = make_float4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<float4*>(t_lo + off) = make_float4(l[0], l[1], l[2], l[3]);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
      tc::wgmma_wait<0>();  // this warpgroup's wgmmas of the previous step (the other stage) are done
      __syncthreads();
      tc::wgmma_fence();
      const uint32_t th = tc::smem_u32(t_hi), tl = tc::smem_u32(t_lo);
#pragma unroll
      for (int ks = 0; ks < KC / 8; ++ks) {
        const uint32_t o = ks * 256u;
#pragma unroll
        for (int j = 0; j < NBLK; ++j) {
          const uint64_t ah = tc::make_smem_desc(th + a_off[j] + o), al = tc::make_smem_desc(tl + a_off[j] + o);
          const uint64_t bh = tc::make_smem_desc(th + b_off[j] + o), bl = tc::make_smem_desc(tl + b_off[j] + o);
          if constexpr (TWO) {
            tc::wgmma_m64n32k8_tf32(acc[j], ah, bh);
            tc::wgmma_m64n32k8_tf32(acc[j], ah, bl);
            tc::wgmma_m64n32k8_tf32(acc[j], al, bh);
          } else {
            tc::wgmma_m64n64k8_tf32(acc[j], ah, bh);
            tc::wgmma_m64n64k8_tf32(acc[j], ah, bl);
            tc::wgmma_m64n64k8_tf32(acc[j], al, bh);
          }
        }
      }
      tc::wgmma_commit();
    }
    tc::wgmma_wait<0>();
    __syncthreads();  // every warpgroup's wgmmas are done: the tiles are about to be overwritten by L

    // ================= accumulators -> B = A + Y^T Y + reg I, fp32, lower triangle, from this warpgroup's blocks
#pragma unroll
    for (int j = 0; j < NBLK; ++j) {
#pragma unroll
      for (int i = 0; i < BW / 2; ++i) {
        const int r = r0[j] + tc::frag_row(i, t), c = c0[j] + tc::frag_col(i, t);
        if (r < f && c <= r) S.L[roff(r) + c] = (float)((double)acc[j][i] + YtY[(size_t)c * f + r] + (r == c ? reg : 0.0));
      }
    }
    if (tid >= 256 && tid - 256 < f) S.rs[tid - 256] = my_rhs;  // the upper half's share of the right-hand side
    __syncthreads();
    if (tid < f) { const double b = my_rhs + S.rs[tid]; S.b0[tid] = b; S.xs[tid] = b; }
    __syncthreads();

    // ================= blocked Cholesky, fp32, in place
    for (int k0 = 0; k0 < f; k0 += NB) {
      const int nb = min(NB, f - k0);
      // ---- diagonal block in the registers of warp 0: lane i holds row i; its inverse for the solves
      if (warp == 0) {
        float a[NB];
        {
          // row k0 + lane, columns k0 .. k0 + 31 (16-byte aligned); entries past the diagonal belong to the next row or to
          // padding and are never used (see below), lanes >= nb read a valid address of the last row
          const float* src = S.L + roff(k0 + min(lane, nb - 1)) + k0;
#pragma unroll
          for (int c4 = 0; c4 < NB / 4; ++c4) {
            const float4 t4 = (c4 * 4 <= lane) ? *reinterpret_cast<const float4*>(src + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            a[c4 * 4 + 0] = t4.x; a[c4 * 4 + 1] = t4.y; a[c4 * 4 + 2] = t4.z; a[c4 * 4 + 3] = t4.w;
          }
        }
        // Lane i holds row i; only the lower triangle (c <= i) of a[] is ever read -- by this lane, or through the shuffles that
        // fetch lane c's a[j] with c > j -- so nothing below is predicated on the lane: the entries above the diagonal hold
        // garbage that feeds only garbage.  One reciprocal square root per step instead of a square root and a division (the
        // factor only has to be fp32-good: the refinement is against the exact operator).
        bool bad = false;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          if (j < nb) {
            const float ajj = __shfl_sync(0xffffffffu, a[j], j);
            bad = bad || !(ajj > 0.f);
            const float rinv = rsqrtf(fmaxf(ajj, 1e-30f));
            if (lane == 0) S.rdiag[j] = rinv;  // 1 / L11[j][j] for the forward substitutions below
            a[j] = (lane == j) ? ajj * rinv : a[j] * rinv;
#pragma unroll
            for (int c = j + 1; c < NB; ++c) a[c] = fmaf(-a[j], __shfl_sync(0xffffffffu, a[j], c), a[c]);
          }
        }
        if (bad && lane == 0) atomicExch(info, row + 1);
        if (lane < nb) {
#pragma unroll
          for (int c = 0; c < NB; ++c)
            if (c <= lane) S.L[roff(k0 + lane) + k0 + c] = a[c];
        }
      }
      __syncthreads();
      const int R0 = k0 + nb;
      // ---- one forward substitution against L11 for 32 + n_below right-hand sides: the rows of the panel below the block
      // (row r of L21 = A21 L11^-T, threads 32..) and, in warp 0, the unit vectors -- column `lane` of inv(L11), kept for the
      // solves.  The inverse costs the critical path nothing: it runs beside the panel.
      {
        const bool is_inv = tid < 32;
        const int r = R0 + tid - 32;
        if (is_inv || r < f) {
          float* Lr = is_inv ? nullptr : S.L + roff(r) + k0;
          float x[NB];
          if (is_inv) {
#pragma unroll
            for (int c = 0; c < NB; ++c) x[c] = (c == lane) ? 1.f : 0.f;
          } else {
#pragma unroll
            for (int c4 = 0; c4 < NB / 4; ++c4) {
              const float4 t4 = *reinterpret_cast<const float4*>(Lr + c4 * 4);
              x[c4 * 4 + 0] = t4.x; x[c4 * 4 + 1] = t4.y; x[c4 * 4 + 2] = t4.z; x[c4 * 4 + 3] = t4.w;
            }
          }
#pragma unroll
          for (int j = 0; j < NB; ++j) {
            if (j < nb) {
              const float* Lj = S.L + roff(k0 + j) + k0;  // same address in every thread: broadcast
              float s = x[j];
#pragma unroll
              for (int c = 0; c < NB; ++c)
                if (c < j) s -= x[c] * Lj[c];
              x[j] = s * S.rdiag[j];
            }
          }
          if (is_inv) {
            float* inv = S.dinv + (k0 / NB) * NB * NBP;
#pragma unroll
            for (int i = 0; i < NB; ++i) inv[i * NBP + lane] = (i >= lane && i < nb && lane < nb) ? x[i] : 0.f;  // inv[i][j] = (L11^-1 e_j)[i]
          } else {
#pragma unroll
            for (int c4 = 0; c4 < NB / 4; ++c4)
              *reinterpret_cast<float4*>(Lr + c4 * 4) = make_float4(x[c4 * 4 + 0], x[c4 * 4 + 1], x[c4 * 4 + 2], x[c4 * 4 + 3]);
          }
        }
      }
      __syncthreads();
      if (R0 >= f) break;
      // ---- trailing update A22 -= L21 L21^T (lower part).  A warp owns a 16-row x 32-column block: lane -> 4 x 4 tile
      // (rows 4 (lane >> 3).., columns 4 (lane & 7)..): the 128-bit loads of a row / column panel are shared by 8 / 4 lanes
      {
        const int nt = f - R0;                    // trailing order
        const int nsr = (nt + 15) / 16;           // 16-row strips; strip si meets (si >> 1) + 1 column strips of 32
        // super-tiles in row-major order of the lower triangle, dealt round-robin to the warps: strips 2a and 2a + 1 start at
        // a (a + 1) and (a + 1)^2
        const int n_super = (nsr & 1) ? ((nsr + 1) / 2) * ((nsr + 1) / 2) : (nsr / 2) * (nsr / 2 + 1);
        for (int n = warp; n < n_super; n += NW) {
          {
            int a = (int)sqrtf((float)n);
            while (a * a > n) --a;
            while ((a + 1) * (a + 1) <= n) ++a;
            int si, sj;
            if (n >= a * (a + 1)) { si = 2 * a; sj = n - a * (a + 1); } else { si = 2 * a - 1; sj = n - a * a; }
            const int r0 = R0 + si * 16 + (lane >> 3) * 4, c0 = R0 + sj * 32 + (lane & 7) * 4;
            if (c0 > r0 + 3 || r0 >= f) continue;
            float acc[4][4];
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
              for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;
#pragma unroll
            for (int kk = 0; kk < NB / 4; ++kk) {
              float4 av[4], bv[4];
#pragma unroll
              for (int x = 0; x < 4; ++x) {
                const int r = min(r0 + x, f - 1), c = min(c0 + x, f - 1);
                av[x] = *reinterpret_cast<const float4*>(S.L + roff(r) + k0 + kk * 4);
                bv[x] = *reinterpret_cast<const float4*>(S.L + roff(c) + k0 + kk * 4);
              }
#pragma unroll
              for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y)
                  acc[x][y] += av[x].x * bv[y].x + av[x].y * bv[y].y + av[x].z * bv[y].z + av[x].w * bv[y].w;
            }
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
              for (int y = 0; y < 4; ++y) {
                const int r = r0 + x, c = c0 + y;
                if (r < f && c <= r) S.L[roff(r) + c] -= acc[x][y];
              }
          }
        }
      }
      __syncthreads();
    }

    // ================= solve and refine
    solve_forward(S, S.xs, f);
    solve_backward(S, S.xs, f);
    for (int it = 0; it < n_refine; ++it) {
      // part[w][m] = sum over this warp's profile entries of (c_k - 1) (y_k . x) y_k[m]; lane owns m = lane + 32 t
      double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll 2
      for (int q = p0 + warp; q < p1; q += NW) {  // two entries' loads in flight
        const double* y = Y + (size_t)idx[q] * f;
        double yv[8], dot = 0.0;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int m = lane + 32 * t;
          yv[t] = m < f ? y[m] : 0.0;
          dot += m < f ? yv[t] * S.xs[m] : 0.0;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, off);
        const double wd = ((double)conf[q] - 1.0) * dot;
#pragma unroll
        for (int t = 0; t < 8; ++t) acc[t] += wd * yv[t];
      }
#pragma unroll
      for (int t = 0; t < 8; ++t)
        if (lane + 32 * t < f) S.part[warp * f + lane + 32 * t] = acc[t];
      __syncthreads();
      if (tid < f) {
        double ax = reg * S.xs[tid];
        for (int w = 0; w < NW; ++w) ax += S.part[w * f + tid];
#pragma unroll 8
        for (int n = 0; n < f; ++n) ax += YtY[(size_t)n * f + tid] * S.xs[n];  // symmetric: coalesced over tid; eight loads in flight
        S.rs[tid] = S.b0[tid] - ax;
      }
      __syncthreads();
      if (warp == 0 && (it == 0 || it == n_refine - 1)) {  // |r|^2 before the first and before the last correction
        double r2 = 0.0, b2 = 0.0;
        for (int m = lane; m < f; m += 32) { r2 += S.rs[m] * S.rs[m]; b2 += S.b0[m] * S.b0[m]; }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) { r2 += __shfl_xor_sync(0xffffffffu, r2, off); b2 += __shfl_xor_sync(0xffffffffu, b2, off); }
        if (lane == 0) {
          if (it == 0) { s_norm[1] = r2; s_norm[2] = b2; }
          if (it == n_refine - 1) s_norm[0] = r2;
        }
      }
      solve_forward(S, S.rs, f);
      solve_backward(S, S.rs, f);
      if (tid < f) S.xs[tid] += S.rs[tid];
      __syncthreads();
    }
    // the residual must have shrunk at least 1000-fold between the first and the last correction (or sit at the rounding floor
    // of the exact operator already); otherwise the fp32 factor is too far from the exact operator for this row
    if (n_refine >= 2 && tid == 0 && !(s_norm[0] <= 1e-3 * s_norm[1] || s_norm[0] <= 1e-22 * s_norm[2])) atomicExch(redo, 1);
    if (tid < f) X[(size_t)row * f + tid] = S.xs[tid];
    __syncthreads();
  }
}

inline size_t smem_bytes(int f) {
  size_t o = std::max<size_t>((size_t)roff(f) * 4, (size_t)STAGES * 2 * TILE);
  o = (o + 127) & ~(size_t)127;
  o += sizeof(double) * (3 * (size_t)f + NW * (size_t)f + KC) + sizeof(float) * ((size_t)((f + NB - 1) / NB) * NB * NBP + KC) + sizeof(int) * KC + sizeof(float) * NB;
  return o + 64;
}

}  // namespace ials2
}  // namespace b200
