// fp32-accurate GEMM on the Hopper tensor cores (wgmma, sm_90a): C = alpha * op(A) * op(B) + beta * C.
//
// Each operand element x is split into two TF32 numbers, x = hi + lo (hi = rna_tf32(x), lo = rna_tf32(x - hi)), and every
// 64 x 128 x 8 step of a warpgroup issues three wgmma.mma_async .tf32 instructions, hi*hi + hi*lo + lo*hi, into one fp32
// accumulator tile held in registers ("3xTF32": the dropped lo*lo term is ~2^-22 relative, so the result is fp32-accurate,
// which the 1e-4 parity bar of the EASE_R inverse needs; a single TF32 pass is not).
//
// One CTA (256 threads = two warpgroups) per 128 x 128 output tile; warpgroup g owns rows 64 g .. 64 g + 63.  K is consumed
// in chunks of 32: all threads load the two operand chunks from global memory, split them and store hi / lo tiles in shared
// memory in the canonical no-swizzle K-major layout (8-row x 16-byte core matrices; LBO = 128 B between K-adjacent cores,
// SBO = 1024 B between 8-row groups), two stages deep.  The loads of chunk k+1 overlap the wgmmas of chunk k: a warpgroup
// waits for its own wgmmas of chunk k before the block-wide barrier that publishes chunk k+1, so once that barrier is passed
// nobody reads the stage chunk k+2 will overwrite.  Descriptor bit layout as cute/arch/mma_sm90_desc.hpp (GmmaDescriptor).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {
namespace tc {

constexpr int BM = 128, BN = 128, BK = 32;   // BK in fp32/tf32 elements (128 bytes per row)
constexpr int TILE_BYTES = BM * BK * 4;      // 16 KB
constexpr int STAGES = 2;
constexpr int SMEM_BYTES = STAGES * 4 * TILE_BYTES;  // {A_hi, A_lo, B_hi, B_lo} per stage
constexpr int THREADS = 256;
constexpr uint32_t WG_ROWS_BYTES = 64 / 8 * (BK / 4) * 128;  // 64 tile rows = 8 row groups of 1024 B

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);                     // start address, 16-byte units
  d |= (uint64_t)((128u >> 4) & 0x3FFFu) << 16;                // leading byte offset: next core matrix along K
  d |= (uint64_t)((((BK / 4) * 128u) >> 4) & 0x3FFFu) << 32;   // stride byte offset: next 8-row group
  return d;                                                    // base offset 0, layout type 0 = no swizzle (interleave)
}

__device__ __forceinline__ uint32_t tile_offset(int row, int k) {
  return (uint32_t)((((row >> 3) * (BK / 4) + (k >> 2)) << 7) + ((row & 7) << 4) + ((k & 3) << 2));
}

__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(x - hi));
  lo = __uint_as_float(l);
}

// tile(row, k) = src[(row0 + row) * ld + k0 + k]   (k contiguous in memory)
__device__ __forceinline__ void load_tile_kcontig(const float* __restrict__ src, long long ld, int row0, int k0,
                                                  unsigned char* hi_tile, unsigned char* lo_tile, int tid) {
#pragma unroll
  for (int e = 0; e < (BM * BK / 4) / THREADS; ++e) {
    const int idx = tid + e * THREADS;
    const int r7 = idx & 7, k4 = (idx >> 3) & 7, m8 = idx >> 6;
    const int row = m8 * 8 + r7;
    const float4 v = *reinterpret_cast<const float4*>(src + (long long)(row0 + row) * ld + k0 + k4 * 4);
    float4 h, l;
    split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
    const uint32_t off = tile_offset(row, k4 * 4);
    *reinterpret_cast<float4*>(hi_tile + off) = h;
    *reinterpret_cast<float4*>(lo_tile + off) = l;
  }
}

// tile(row, k) = src[(k0 + k) * ld + row0 + row]   (row contiguous in memory)
__device__ __forceinline__ void load_tile_rowcontig(const float* __restrict__ src, long long ld, int row0, int k0,
                                                    unsigned char* hi_tile, unsigned char* lo_tile, int tid) {
#pragma unroll
  for (int e = 0; e < (BM * BK / 4) / THREADS; ++e) {
    const int idx = tid + e * THREADS;
    const int m4 = idx & 31, k = idx >> 5;  // 32 float4 along the rows, 32 values of k
    const float4 v = *reinterpret_cast<const float4*>(src + (long long)(k0 + k) * ld + row0 + m4 * 4);
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float h, l;
      split_tf32(x[c], h, l);
      const uint32_t off = tile_offset(m4 * 4 + c, k);
      *reinterpret_cast<float*>(hi_tile + off) = h;
      *reinterpret_cast<float*>(lo_tile + off) = l;
    }
  }
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE;\n"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// ---- warpgroup MMA (every thread of the warpgroup executes these)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D(64 x 128) += A(64 x 8) B(128 x 8)^T: tf32 operands K-major in shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}

// D(64 x 64) += A(64 x 8) B(64 x 8)^T: tf32 operands K-major in shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}

// D(64 x 32) += A(64 x 8) B(32 x 8)^T: tf32 operands K-major in shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}

// Accumulator fragment of a 64 x N wgmma tile: register i of thread t (warp w = (t / 32) % 4, lane l) holds
// row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
__device__ __forceinline__ int frag_row(int i, int t) { return 16 * ((t >> 5) & 3) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int t) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// TA: op(A)(m, k) = A[k * lda + m]; TB: op(B)(k, n) = B[n * ldb + k].  TRI: op(A) = L^T, op(B) = L with L lower
// triangular, so only k >= max(m0, n0) contributes.  M, N multiples of 128, K a multiple of 32.  blockIdx.z = batch.
template <bool TA, bool TB, bool TRI>
__global__ void __launch_bounds__(THREADS, 1) tc_gemm_kernel(int M, int N, int K, float alpha, const float* __restrict__ A, int lda,
                                                             long long strideA, const float* __restrict__ B, int ldb, long long strideB,
                                                             float beta, float* C, int ldc, long long strideC) {
  extern __shared__ __align__(1024) unsigned char smem[];
  A += (long long)blockIdx.z * strideA;
  B += (long long)blockIdx.z * strideB;
  C += (long long)blockIdx.z * strideC;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tid = threadIdx.x, wg = tid >> 7;
  unsigned char* tiles = smem;

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  const int k_begin = TRI ? (max(m0, n0) / BK) * BK : 0;
  const int nk = (K - k_begin) / BK;
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb & 1;
    const int k0 = k_begin + kb * BK;
    unsigned char* a_hi = tiles + (s * 4 + 0) * TILE_BYTES;
    unsigned char* a_lo = tiles + (s * 4 + 1) * TILE_BYTES;
    unsigned char* b_hi = tiles + (s * 4 + 2) * TILE_BYTES;
    unsigned char* b_lo = tiles + (s * 4 + 3) * TILE_BYTES;
    if (TA) load_tile_rowcontig(A, lda, m0, k0, a_hi, a_lo, tid); else load_tile_kcontig(A, lda, m0, k0, a_hi, a_lo, tid);
    if (TB) load_tile_kcontig(B, ldb, n0, k0, b_hi, b_lo, tid); else load_tile_rowcontig(B, ldb, n0, k0, b_hi, b_lo, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
    wgmma_wait<0>();  // this warpgroup's wgmmas of chunk kb-1 (the other stage) are done
    __syncthreads();
    wgmma_fence();
    const uint32_t ah = smem_u32(a_hi) + wg * WG_ROWS_BYTES, al = smem_u32(a_lo) + wg * WG_ROWS_BYTES;
    const uint32_t bh = smem_u32(b_hi), bl = smem_u32(b_lo);
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {  // one wgmma consumes K = 8 tf32 = two core matrices = 256 bytes
      const uint32_t o = ks * 256u;
      wgmma_m64n128k8_tf32(acc, make_smem_desc(ah + o), make_smem_desc(bh + o));
      wgmma_m64n128k8_tf32(acc, make_smem_desc(ah + o), make_smem_desc(bl + o));
      wgmma_m64n128k8_tf32(acc, make_smem_desc(al + o), make_smem_desc(bh + o));
    }
    wgmma_commit();
  }
  wgmma_wait<0>();

  // epilogue: every thread writes its accumulator fragment, two adjacent columns per store
  const int t = tid & 127;
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    float2* dst = reinterpret_cast<float2*>(C + (long long)(m0 + wg * 64 + frag_row(i, t)) * ldc + n0 + frag_col(i, t));
    float2 o = make_float2(alpha * acc[i], alpha * acc[i + 1]);
    if (beta != 0.f) {
      const float2 old = *dst;
      o.x += beta * old.x; o.y += beta * old.y;
    }
    *dst = o;
  }
}

}  // namespace tc
}  // namespace b200
