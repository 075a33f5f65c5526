// Development: what one GPU sustains on the access pattern of the K1-D upper pass's gather (csrc/sim_k1d.cuh), without its
// shared-memory atomics: every warp reads batches of 32 random, 16-byte aligned segments of SEG bytes from a buffer far
// larger than L2 as one stream of 16-byte chunks, STEPS loads of 32 chunks in flight, 256 threads per CTA and four CTAs per
// SM (held there by 50 KB of dynamic shared memory, the upper pass's counters at 200 K columns), and sums what it reads.
// Prints one JSON line per segment size; GB/s counts the segment bytes only (the sectors a misaligned segment drags in are
// not counted).  Built and run by tools/dev_gather_bw.py.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int THREADS = 256, CTAS = 4, STEPS = 4, SMEM = 50 * 1024;

__device__ __forceinline__ unsigned mix(unsigned x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

__global__ void __launch_bounds__(THREADS, CTAS) gather_kernel(const int4* __restrict__ buf, unsigned n_chunks, int seg_chunks, int batches,
                                                               unsigned long long* out) {
  extern __shared__ unsigned smem[];
  const int lane = threadIdx.x & 31;
  const unsigned gwarp = (blockIdx.x * THREADS + threadIdx.x) >> 5;
  const int total = 32 * seg_chunks;  // chunks of a batch
  unsigned sum = 0u;
  for (int b = 0; b < batches; ++b) {
    // lane r holds the start of segment r of this batch
    const unsigned start = mix(gwarp * 0x9e3779b9U + (unsigned)b * 32u + (unsigned)lane) % (n_chunks - (unsigned)seg_chunks);
    for (int b0 = 0; b0 < total; b0 += 32 * STEPS) {
      int4 v[STEPS];
#pragma unroll
      for (int q = 0; q < STEPS; ++q) {
        const int f = b0 + 32 * q + lane, row = (f / seg_chunks) & 31;
        const unsigned rs = __shfl_sync(0xffffffffu, start, row);
        if (f < total) v[q] = __ldg(buf + rs + (f - row * seg_chunks));
      }
#pragma unroll
      for (int q = 0; q < STEPS; ++q)
        if (b0 + 32 * q + lane < total) sum += (unsigned)(v[q].x + v[q].y + v[q].z + v[q].w);
    }
  }
  if (sum == 0x12345678u) smem[threadIdx.x] = sum;  // keeps the shared memory and the loads alive
  atomicAdd(out, (unsigned long long)sum);
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const size_t bytes = 2ull << 30;
  const unsigned n_chunks = (unsigned)(bytes / 16);
  int4* buf;
  unsigned long long* out;
  CK(cudaMalloc(&buf, bytes));
  CK(cudaMalloc(&out, 8));
  CK(cudaMemset(buf, 1, bytes));
  CK(cudaMemset(out, 0, 8));
  CK(cudaFuncSetAttribute(gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  CK(cudaFuncSetAttribute(gather_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
  int resident = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, gather_kernel, THREADS, SMEM));
  const int grid = prop.multiProcessorCount * CTAS;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const int segs[2] = {208, 128};
  for (int s = 0; s < 2; ++s) {
    const int seg_chunks = segs[s] / 16;
    const int batches = 600;  // per warp: 4 224 warps x 600 x 32 segments = 81 M segments, 10 to 17 GB
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {  // the first one warms up
      CK(cudaEventRecord(e0));
      gather_kernel<<<grid, THREADS, SMEM>>>(buf, n_chunks, seg_chunks, batches, out);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaGetLastError());
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rep > 0 && ms < best) best = ms;
    }
    const double gb = (double)grid * (THREADS / 32) * batches * 32.0 * segs[s] / 1e9;
    printf("{\"device\": \"%s\", \"sms\": %d, \"ctas_per_sm_resident\": %d, \"segment_bytes\": %d, \"gb\": %.2f, \"ms_best_of_3\": %.3f, \"gb_per_s\": %.0f}\n",
           prop.name, prop.multiProcessorCount, resident, segs[s], gb, best, gb / (best * 1e-3));
  }
  CK(cudaFree(buf));
  CK(cudaFree(out));
  return 0;
}
