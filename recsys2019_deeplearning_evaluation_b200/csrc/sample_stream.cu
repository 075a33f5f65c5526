// SampleStream (sampler.cuh): an SGD trainer's epoch of samples in device arrays, from the host glibc replay, the glibc
// stream resolved on the device, or Philox on the device.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "sampler.cuh"

namespace b200 {
namespace {

// The Philox stream of the users [user_lo, user_lo + n_users); c3 tells the trainers' streams apart
__global__ void philox_sample_kernel(const int* __restrict__ indptr, const int* __restrict__ indices, const float* __restrict__ data,
                                     int user_lo, int n_users, int n_items, bool bpr, float quota, long long n_samples, unsigned seed,
                                     unsigned epoch, unsigned c3, int* su, int* si, int* sj, float* sr) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_samples) return;
  PhiloxDraws d{(unsigned long long)g, seed, epoch, c3};
  Sample s;
  draw_sample(d, indptr, indices, data, user_lo, n_users, n_items, bpr, quota, s);
  su[g] = s.u;
  si[g] = s.i;
  if (bpr) sj[g] = s.j; else sr[g] = s.r;
}

// =====================================================================================================================
// glibc stream on the device.  The reference draws its samples with libc rand() (sampleBPR_Cython pyx:943-987,
// sampleMSE_Cython :881-938): a sequential recurrence feeding rejection loops, so sample g's first draw depends on how many
// draws every earlier sample consumed.  The raw stream itself is cheap to produce in order (1 ns per draw on the host);
// what made the host replay slow (160 ms per C5 epoch) are the dependent memory lookups of the acceptance rules.  Here:
//   1. the host appends raw draws to a pinned buffer and uploads them;
//   2. glibc_len_kernel: for EVERY position p of the buffer, how many draws a sample STARTING at p would consume;
//   3. pointer doubling: J_0[p] = p + len[p], J_{k+1} = J_k o J_k, so that any number of samples can be skipped at once;
//   4. glibc_emit_kernel: sample g starts where the binary expansion of g leads from position 0; it is re-evaluated there
//      and written out.  The number of draws the epoch consumed tells the host where the next epoch's stream begins.
// Bit-identical to the host replay (same draws, same rules); tests compare the two.
struct GlibcView {
  const int* __restrict__ raw; int R;  // draws raw[0 .. R)
  const int* __restrict__ indptr; const int* __restrict__ indices; const float* __restrict__ data;
  int n_users, n_items; bool bpr; float quota;
};

// the sample starting at raw position p: returns the position after its last draw (> R when the buffer ran out)
__device__ __forceinline__ int glibc_sample_at(const GlibcView& v, int p, Sample* out) {
  GlibcReplay d{v.raw, p, v.R};
  Sample s{};
  if (!draw_sample(d, v.indptr, v.indices, v.data, 0, v.n_users, v.n_items, v.bpr, v.quota, s)) return v.R + 1;
  if (out) *out = s;
  return d.q;
}

__global__ void glibc_len_kernel(const GlibcView v, int* __restrict__ nxt) {  // nxt[p] = start of the following sample; nxt[R] = R
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > v.R) return;
  nxt[p] = p == v.R ? v.R : min(glibc_sample_at(v, p, nullptr), v.R);
}

__global__ void glibc_double_kernel(const int* __restrict__ jk, int R, int* __restrict__ jk1) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p <= R) jk1[p] = jk[jk[p]];
}

// sample g: follow the binary expansion of g through the jump tables (tables[k] = J_k, (R + 1) ints each), evaluate, store
__global__ void glibc_emit_kernel(const GlibcView v, const int* __restrict__ tables, int levels, long long n_samples, int* su, int* si,
                                  int* sj, float* sr, int* consumed) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_samples) return;
  int p = 0;
  for (int k = 0; k < levels; ++k)
    if ((g >> k) & 1) p = tables[(size_t)k * (v.R + 1) + p];
  Sample s{};
  const int q = p < v.R ? glibc_sample_at(v, p, &s) : v.R + 1;
  su[g] = s.u; si[g] = s.i;
  if (v.bpr) sj[g] = s.j; else sr[g] = s.r;
  if (q > v.R) atomicMax(consumed, 0x7FFFFFFF);  // the buffer ran out somewhere: the host extends it and repeats
  else if (g == n_samples - 1) atomicMax(consumed, q);
}

}  // namespace

SampleStream::~SampleStream() {
  if (h_raw) cudaFreeHost(h_raw);
}

void SampleStream::init(int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_ip, const int32_t* h_ix, const float* h_d,
                        bool bpr_, double quota_, size_t capacity, bool philox_, unsigned c3_, unsigned glibc_seed, bool glibc_device_) {
  n_users_ = (int)n_users; n_items_ = (int)n_items;
  bpr = bpr_; quota = quota_; philox = philox_; c3 = c3_;
  glibc_device = glibc_device_;
  if (const char* e = getenv("B200REC_GLIBC_HOST")) glibc_device = glibc_device && atoi(e) == 0;
  rng.seed(glibc_seed);
  h_indptr.assign(h_ip, h_ip + n_users + 1);
  h_indices.assign(h_ix, h_ix + nnz);
  if (!bpr) h_data.assign(h_d, h_d + nnz);
  indptr.alloc((size_t)n_users + 1);
  indices.alloc((size_t)std::max<int64_t>(nnz, 1));
  B200_CUDA(cudaMemcpy(indptr.get(), h_ip, sizeof(int) * ((size_t)n_users + 1), cudaMemcpyHostToDevice));
  if (nnz) B200_CUDA(cudaMemcpy(indices.get(), h_ix, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice));
  if (!bpr && (philox || glibc_device)) {
    data.alloc((size_t)std::max<int64_t>(nnz, 1));
    if (nnz) B200_CUDA(cudaMemcpy(data.get(), h_d, sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice));
  }
  su.alloc(capacity); si.alloc(capacity);
  if (bpr) sj.alloc(capacity); else sr.alloc(capacity);
}

void SampleStream::draw_glibc(long long n, cudaStream_t st) {
  if (philox) return;
  host_drawn = !(glibc_device && n * 4 + 65536 < (1ll << 30));
  if (!host_drawn) {
    glibc_device_samples(n, st);
  } else {
    hs.draw(rng, h_indptr.data(), h_indices.data(), h_data.data(), n_users_, n_items_, bpr, quota, n);
    B200_CUDA(cudaMemcpyAsync(su.get(), hs.u.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(si.get(), hs.i.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    if (bpr) B200_CUDA(cudaMemcpyAsync(sj.get(), hs.j.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    else B200_CUDA(cudaMemcpyAsync(sr.get(), hs.r.data(), sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, st));
  }
  drawn = n;
}

void SampleStream::draw_philox(long long n, unsigned seed, unsigned epoch, int user_lo, int n_users, cudaStream_t st) {
  if (!philox) return;
  philox_sample_kernel<<<div_up(n, 256), 256, 0, st>>>(indptr.get(), indices.get(), data.get(), user_lo, n_users, n_items_, bpr,
                                                       (float)quota, n, seed, epoch, c3, su.get(), si.get(), sj.get(), sr.get());
  B200_CUDA(cudaGetLastError());
  count_launch();
  drawn = n;
}

void SampleStream::copy_out(int* u, int* i, int* j, float* r) const {
  B200_CUDA(cudaDeviceSynchronize());
  const size_t n = (size_t)drawn;
  if (u) B200_CUDA(cudaMemcpy(u, su.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
  if (i) B200_CUDA(cudaMemcpy(i, si.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
  if (j && bpr) B200_CUDA(cudaMemcpy(j, sj.get(), sizeof(int) * n, cudaMemcpyDeviceToHost));
  if (r && !bpr) B200_CUDA(cudaMemcpy(r, sr.get(), sizeof(float) * n, cudaMemcpyDeviceToHost));
}

// The n samples from the glibc stream, resolved on the device (see glibc_len_kernel).  Synchronises the stream once (the
// host must know how many draws were consumed before it can continue the stream).
void SampleStream::glibc_device_samples(long long n, cudaStream_t st) {
  const int per = 3;  // draws of a sample without rejections (user, positive | quota, negative | item)
  int levels = 1;
  while ((1ll << levels) < n) ++levels;
  long long want = n * per + n / 16 + 4096;
  for (int attempt = 0;; ++attempt) {
    B200_REQUIRE(attempt < 8 && want < (1ll << 30), "the glibc replay buffer does not converge (degenerate URM?)");
    if (want > raw_cap) {
      int* fresh = nullptr;
      B200_CUDA(cudaMallocHost(reinterpret_cast<void**>(&fresh), sizeof(int) * (size_t)want));
      if (raw_have) memcpy(fresh, h_raw, sizeof(int) * (size_t)raw_have);
      if (h_raw) cudaFreeHost(h_raw);
      h_raw = fresh;
      raw_cap = want;
      d_raw.alloc((size_t)want);
    }
    for (long long q = raw_have; q < want; ++q) h_raw[q] = rng.next();
    raw_have = want;
    const int R = (int)want;
    if ((long long)levels * (R + 1) > tables_cap) {
      tables_cap = (long long)levels * (R + 1);
      d_tables.alloc((size_t)tables_cap);
    }
    if (d_consumed.n == 0) d_consumed.alloc(1);
    B200_CUDA(cudaMemcpyAsync(d_raw.get(), h_raw, sizeof(int) * (size_t)R, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemsetAsync(d_consumed.get(), 0, sizeof(int), st));
    GlibcView v{d_raw.get(), R, indptr.get(), indices.get(), data.get(), n_users_, n_items_, bpr, (float)quota};
    int* T = d_tables.get();
    glibc_len_kernel<<<div_up(R + 1, 256), 256, 0, st>>>(v, T);
    for (int k = 0; k + 1 < levels; ++k)
      glibc_double_kernel<<<div_up(R + 1, 256), 256, 0, st>>>(T + (size_t)k * (R + 1), R, T + (size_t)(k + 1) * (R + 1));
    glibc_emit_kernel<<<div_up(n, 256), 256, 0, st>>>(v, T, levels, n, su.get(), si.get(), sj.get(), sr.get(), d_consumed.get());
    B200_CUDA(cudaGetLastError());
    count_launch(levels + 1);
    int consumed = 0;
    B200_CUDA(cudaMemcpyAsync(&consumed, d_consumed.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (consumed != 0x7FFFFFFF && consumed <= R) {
      // the unread tail opens the next epoch's stream
      raw_have = R - consumed;
      if (raw_have) memmove(h_raw, h_raw + consumed, sizeof(int) * (size_t)raw_have);
      return;
    }
    want = want + want / 2;  // many rejections (dense profiles): a longer buffer, same draws in front
  }
}

}  // namespace b200
