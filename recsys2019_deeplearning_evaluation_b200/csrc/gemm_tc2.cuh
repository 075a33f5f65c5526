// Second-generation 3xTF32 wgmma GEMM (sm_90a): pre-packed operands fed by the TMA engine's bulk copies.
//
// gemm_tc.cuh spends most of its time converting operands (cvt.rna.tf32) and storing them transposed with 4-byte stores,
// and the loads of chunk k+1 only start after the whole block has synchronised on chunk k.  Here
//   * a pack pass splits every operand ONCE into hi / lo TF32 parts and writes them in the exact shared-memory image of a
//     128 x 32 wgmma tile (canonical no-swizzle K-major layout, same tile_offset as gemm_tc.cuh), hi and lo adjacent:
//     packed[(row_block * KC + k_chunk) * 8192 floats] = {hi tile 16 KB, lo tile 16 KB};
//   * the GEMM kernel is warp-specialised: one producer lane (warpgroup 0) issues two 32 KB `cp.async.bulk` copies per
//     128x128x32 step (A hi+lo, B hi+lo) that complete on the stage's "full" mbarrier; each of the two consumer warpgroups
//     waits for it, issues the 12 wgmmas of its 64 x 128 half of the step (hi*hi + hi*lo + lo*hi) and, once the wgmmas of
//     the step before have completed, releases that step's stage on its "empty" mbarrier; three stages deep (192 KB), no
//     block-wide barrier at all;
//   * each consumer warpgroup writes its accumulators from registers (the epilogue of gemm_tc.cuh).
// O(M K + N K) pack work against O(M N K) MMA work; the packed copies live in a workspace the caller provides.
#pragma once
#include "gemm_tc.cuh"

namespace b200 {
namespace tc2 {

using tc::BK;
using tc::BM;
using tc::BN;
using tc::TILE_BYTES;
constexpr int STAGES = 3;
constexpr int STAGE_BYTES = 4 * TILE_BYTES;                  // A hi, A lo, B hi, B lo
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 64;        // + full[3], empty[3] barriers
constexpr int THREADS = 256;                                 // pack kernel
constexpr int GEMM_THREADS = 384;                            // producer warpgroup + two consumer warpgroups
constexpr int PAIR_FLOATS = 2 * TILE_BYTES / 4;              // one packed (hi, lo) tile pair: 8192 floats

// One CTA packs one 128 x 32 tile of op(X): KCONTIG = the k index is contiguous in memory (tile(row, k) = src[row*ld + k]),
// otherwise the row index is (tile(row, k) = src[k*ld + row]).  grid = (K/32, R/128, batch).
template <bool KCONTIG>
__global__ void __launch_bounds__(THREADS) pack_tiles_kernel(const float* __restrict__ src, int ld, long long stride_batch,
                                                             float* __restrict__ dst, long long dst_stride_batch) {
  extern __shared__ __align__(16) unsigned char sm[];  // 2 * TILE_BYTES
  const int kc = blockIdx.x, rb = blockIdx.y, tid = threadIdx.x;
  const int KC = gridDim.x;
  src += (long long)blockIdx.z * stride_batch;
  if (KCONTIG) tc::load_tile_kcontig(src, ld, rb * BM, kc * BK, sm, sm + TILE_BYTES, tid);
  else tc::load_tile_rowcontig(src, ld, rb * BM, kc * BK, sm, sm + TILE_BYTES, tid);
  __syncthreads();
  float4* out = reinterpret_cast<float4*>(dst + (long long)blockIdx.z * dst_stride_batch + ((long long)rb * KC + kc) * PAIR_FLOATS);
  const float4* in = reinterpret_cast<const float4*>(sm);
  for (int i = tid; i < PAIR_FLOATS / 4; i += THREADS) out[i] = in[i];
}

__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}

// C = alpha * op(A) op(B) + beta * C from packed operands.  TRI: only k >= max(m0, n0) contributes (L^T L products).
// grid = (N/128, M/128, batch).
__global__ void __launch_bounds__(GEMM_THREADS, 1) tc2_gemm_kernel(int K, int tri, float alpha, const float* __restrict__ Ap,
                                                                   long long strideAp, const float* __restrict__ Bp, long long strideBp,
                                                                   float beta, float* C, int ldc, long long strideC) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const int mb = blockIdx.y, nb = blockIdx.x;
  const int m0 = mb * BM, n0 = nb * BN;
  const int KC = K / BK;
  Ap += (long long)blockIdx.z * strideAp + (long long)mb * KC * PAIR_FLOATS;
  Bp += (long long)blockIdx.z * strideBp + (long long)nb * KC * PAIR_FLOATS;
  C += (long long)blockIdx.z * strideC;
  const uint32_t tiles = tc::smem_u32(smem);
  const uint32_t bar0 = tiles + STAGES * STAGE_BYTES;  // full[s] = bar0 + 8 s, empty[s] = bar0 + 8 (STAGES + s)

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8u * s) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 2;" ::"r"(bar0 + 8u * (STAGES + s)) : "memory");  // one arrival per consumer
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int kc_begin = tri ? max(m0, n0) / BK : 0;
  const int nk = KC - kc_begin;

  if (wg == 0) {
    if (tid == 0) {  // ---- producer: two 32 KB bulk copies per stage
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % STAGES, it = kb / STAGES;
        if (it > 0) tc::mbar_wait(bar0 + 8u * (STAGES + s), (uint32_t)((it - 1) & 1));  // the wgmmas that read this stage are done
        const uint32_t full = bar0 + 8u * s;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"((uint32_t)STAGE_BYTES) : "memory");
        const uint32_t dst = tiles + (uint32_t)s * STAGE_BYTES;
        bulk_g2s(dst, Ap + (long long)(kc_begin + kb) * PAIR_FLOATS, 2 * TILE_BYTES, full);
        bulk_g2s(dst + 2 * TILE_BYTES, Bp + (long long)(kc_begin + kb) * PAIR_FLOATS, 2 * TILE_BYTES, full);
      }
    }
    return;
  }

  // ---- consumers: warpgroup 1 + h computes rows 64 h .. 64 h + 63 of the tile
  const int h = wg - 1, t = tid & 127;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb % STAGES, it = kb / STAGES;
    tc::mbar_wait(bar0 + 8u * s, (uint32_t)(it & 1));  // both copies of this stage have landed
    const uint32_t ah = tiles + (uint32_t)s * STAGE_BYTES, al = ah + TILE_BYTES, bh = ah + 2 * TILE_BYTES, bl = ah + 3 * TILE_BYTES;
    const uint32_t ra = (uint32_t)h * tc::WG_ROWS_BYTES;
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {  // one wgmma consumes K = 8 tf32 = two core matrices = 256 bytes
      const uint32_t o = ks * 256u;
      tc::wgmma_m64n128k8_tf32(acc, tc::make_smem_desc(ah + ra + o), tc::make_smem_desc(bh + o));
      tc::wgmma_m64n128k8_tf32(acc, tc::make_smem_desc(ah + ra + o), tc::make_smem_desc(bl + o));
      tc::wgmma_m64n128k8_tf32(acc, tc::make_smem_desc(al + ra + o), tc::make_smem_desc(bh + o));
    }
    tc::wgmma_commit();
    tc::wgmma_wait<1>();  // the wgmmas of step kb - 1 are done: its stage may be refilled
    if (kb > 0 && t == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar0 + 8u * (STAGES + (kb - 1) % STAGES)) : "memory");
  }
  tc::wgmma_wait<0>();

#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    float2* dst = reinterpret_cast<float2*>(C + (long long)(m0 + h * 64 + tc::frag_row(i, t)) * ldc + n0 + tc::frag_col(i, t));
    float2 o = make_float2(alpha * acc[i], alpha * acc[i + 1]);
    if (beta != 0.f) {
      const float2 old = *dst;
      o.x += beta * old.x; o.y += beta * old.y;
    }
    *dst = o;
  }
}

}  // namespace tc2
}  // namespace b200
