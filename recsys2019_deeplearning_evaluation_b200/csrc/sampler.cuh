// How an SGD trainer draws a sample: the reference's sampling rule and the random streams that feed it.  The BPR-MF /
// FunkSVD (mf_sgd.cu), SLIM-BPR (slim_bpr.cu) and AsySVD (asysvd.cu) trainers all draw through draw_sample.
//   MatrixFactorization_Cython_Epoch.pyx: sampleMSE_Cython :881-938, sampleBPR_Cython :943-987
//   SLIM_BPR_Cython_Epoch.pyx: sampleBPR_Cython :436-480
// Streams: glibc's rand() replayed on the host (GlibcRandHost) or resolved on the device from uploaded draws (GlibcReplay),
// both draw for draw the reference's; Philox4x32-10 on the device (PhiloxDraws).  SampleStream turns them into an epoch's
// device samples.  tests/test_sample_streams_gpu.py pins every stream value for value.
#pragma once
#include <vector>

#include "common.cuh"

namespace b200 {

struct Sample {
  int u, i, j;  // j: the negative of a BPR sample
  float r;      // the rating of an MSE sample (0 for a negative)
};

// The reference's rule over a draw source: the user (user_lo + draw % n_users) is redrawn until 0 < profile length <
// n_items; an MSE sample with a non-zero quota spends one draw on "positive if uniform <= quota"; a positive is a draw of a
// position in the profile; a negative is redrawn until a binary search does not find it in the (sorted) profile.  Every
// modulo is unsigned 32-bit.  The source gives next() (a raw draw), uniform_le(draw, quota) and empty(); returns false,
// with `out` incomplete, when the source ran out (only GlibcReplay can).  The pragma lets the host-only source GlibcRandHost
// be used from this __host__ __device__ template.
#pragma nv_exec_check_disable
template <class Src>
__host__ __device__ __forceinline__ bool draw_sample(Src& src, const int* indptr, const int* indices, const float* data, int user_lo,
                                                     int n_users, int n_items, bool bpr, double quota, Sample& out) {
  int s, n;
  do {
    if (src.empty()) return false;
    out.u = user_lo + (int)(src.next() % (unsigned)n_users);
    s = indptr[out.u];
    n = indptr[out.u + 1] - s;
  } while (n == 0 || n == n_items);
  bool positive = true;
  if (!bpr && quota != 0.0) {
    if (src.empty()) return false;
    positive = Src::uniform_le(src.next(), quota);
  }
  if (bpr || positive) {
    if (src.empty()) return false;
    const int k = s + (int)(src.next() % (unsigned)n);
    out.i = indices[k];
    if (!bpr) out.r = data[k];
  }
  if (bpr || !positive) {
    int neg;
    for (;;) {
      if (src.empty()) return false;
      neg = (int)(src.next() % (unsigned)n_items);
      int lo = 0, hi = n;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (indices[s + mid] < neg) lo = mid + 1; else hi = mid; }
      if (lo == n || indices[s + lo] != neg) break;
    }
    if (bpr) out.j = neg; else { out.i = neg; out.r = 0.f; }
  }
  return true;
}

// Whether a user in [lo, hi) has 0 < profile length < n_items: draw_sample redraws the user until one does, so on a range
// without such a user a stream that never runs out would never finish a sample.
inline bool has_sampleable_user(const int32_t* h_indptr, int64_t lo, int64_t hi, int64_t n_items) {
  for (int64_t u = lo; u < hi; ++u) {
    const int64_t n = (int64_t)h_indptr[u + 1] - h_indptr[u];
    if (n > 0 && n < n_items) return true;
  }
  return false;
}

// ---- glibc: the reference's rand() stream.  uniform_le is the reference's `rand() <= quota * RAND_MAX` (pyx:901).
__host__ __device__ __forceinline__ bool glibc_uniform_le(unsigned x, double quota) { return (double)x <= quota * 2147483647.0; }

// Host replay of glibc's srand(seed) / rand() (TYPE_3 additive feedback, r[i] = r[i-31] + r[i-3], 310 discarded, >> 1):
// next() is rand().
struct GlibcRandHost {
  int32_t r[31];
  int f = 3, b = 0;
  void seed(unsigned s) {
    int32_t word = s == 0 ? 1 : (int32_t)s;
    r[0] = word;
    for (int i = 1; i < 31; ++i) {
      const long hi = word / 127773, lo = word % 127773;
      long w = 16807 * lo - 2836 * hi;
      if (w < 0) w += 2147483647;
      word = (int32_t)w;
      r[i] = word;
    }
    f = 3; b = 0;
    for (int i = 0; i < 310; ++i) raw();
  }
  uint32_t raw() {
    const uint32_t v = (uint32_t)r[f] + (uint32_t)r[b];
    r[f] = (int32_t)v;
    if (++f == 31) f = 0;  // not `% 31`: the device replay appends millions of draws per epoch on the host
    if (++b == 31) b = 0;
    return v;
  }
  int next() { return (int)(raw() >> 1); }
  bool empty() const { return false; }
  static bool uniform_le(unsigned x, double quota) { return glibc_uniform_le(x, quota); }
};

// rand() values raw[q .. R) uploaded to the device; runs out at R
struct GlibcReplay {
  const int* raw;
  int q, R;
  __device__ bool empty() const { return q >= R; }
  __device__ unsigned next() { return (unsigned)raw[q++]; }
  __device__ static bool uniform_le(unsigned x, double quota) { return glibc_uniform_le(x, quota); }
};

// An epoch's samples drawn on the host from the glibc stream: (u, i, j) for BPR, (u, i, r) for MSE
struct HostSamples {
  std::vector<int> u, i, j;
  std::vector<float> r;
  void draw(GlibcRandHost& rng, const int* indptr, const int* indices, const float* data, int n_users, int n_items, bool bpr,
            double quota, long long n) {
    u.resize((size_t)n); i.resize((size_t)n);
    if (bpr) j.resize((size_t)n); else r.resize((size_t)n);
    Sample s;
    for (size_t g = 0; g < (size_t)n; ++g) {
      draw_sample(rng, indptr, indices, data, 0, n_users, n_items, bpr, quota, s);
      u[g] = s.u; i[g] = s.i;
      if (bpr) j[g] = s.j; else r[g] = s.r;
    }
  }
};

// ---- Philox4x32-10 (Salmon et al., SC'11; the Random123 constants)
__device__ __forceinline__ void philox_round(unsigned& c0, unsigned& c1, unsigned& c2, unsigned& c3, unsigned k0, unsigned k1) {
  const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
  const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
  c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
}

// The draws of sample `idx`: counter (idx low word, idx high word, draw block, c3), key (seed, epoch), the four words of a
// block taken x, y, z, w.  c3 tells the trainers' streams apart.  uniform_le compares the draw's top 24 bits in fp32.
struct PhiloxDraws {
  unsigned long long idx;
  unsigned seed, epoch, c3, blk = 0;
  uint4 cur;
  int pos = 4;
  __device__ bool empty() const { return false; }
  __device__ unsigned next() {
    if (pos == 4) {
      unsigned c0 = (unsigned)idx, c1 = (unsigned)(idx >> 32), c2 = blk++, c3w = c3, k0 = seed, k1 = epoch;
#pragma unroll
      for (int r = 0; r < 10; ++r) { philox_round(c0, c1, c2, c3w, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
      cur = make_uint4(c0, c1, c2, c3w);
      pos = 0;
    }
    const unsigned v = pos == 0 ? cur.x : (pos == 1 ? cur.y : (pos == 2 ? cur.z : cur.w));
    ++pos;
    return v;
  }
  __device__ static bool uniform_le(unsigned x, double quota) { return (float)(x >> 8) * (1.f / 16777216.f) <= (float)quota; }
};

// ---- One trainer's sample stream (sample_stream.cu): the URM it draws from, the epoch's sample buffers and the source that
// fills them.  A glibc stream is drawn before the epoch's timed window (draw_glibc): replayed on the host and uploaded, or
// resolved on the device from uploaded raw draws (glibc_len_kernel).  A Philox stream is drawn inside it (draw_philox).
struct SampleStream {
  bool bpr = true, philox = false;
  double quota = 0.0;                    // MSE: the probability of a positive
  unsigned c3 = 0;                       // Philox: the fourth counter word (PhiloxDraws)
  std::vector<int> h_indptr, h_indices;  // host copy: the host replay and has_sampleable_user read it
  std::vector<float> h_data;             // MSE only
  DevBuf<int> indptr, indices;
  DevBuf<float> data;                    // MSE streams that can draw on the device only
  DevBuf<int> su, si, sj;                // the drawn samples: (u, i, j) for BPR, (u, i, r) for MSE
  DevBuf<float> sr;
  long long drawn = 0;                   // samples of the last draw

  SampleStream() = default;
  SampleStream(const SampleStream&) = delete;
  SampleStream& operator=(const SampleStream&) = delete;
  ~SampleStream();
  // capacity: the most samples one draw makes.  glibc_device: resolve the glibc stream on the device while it fits 32-bit
  // positions (B200REC_GLIBC_HOST=1 forces the host replay: A/B runs, tests).
  void init(int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* indptr, const int32_t* indices, const float* data,
            bool bpr, double quota, size_t capacity, bool philox, unsigned c3, unsigned glibc_seed, bool glibc_device);
  void draw_glibc(long long n, cudaStream_t st);  // nothing on a Philox stream
  // users from [user_lo, user_lo + n_users), Philox key (seed, epoch); nothing on a glibc stream
  void draw_philox(long long n, unsigned seed, unsigned epoch, int user_lo, int n_users, cudaStream_t st);
  // the last draw was the host replay, whose vectors may still be uploading: the epoch synchronises before the next draw
  bool host_vectors_in_flight() const { return host_drawn; }
  void copy_out(int* u, int* i, int* j, float* r) const;  // the last draw (null: skipped); synchronises the device

 private:
  int n_users_ = 0, n_items_ = 0;
  bool glibc_device = false, host_drawn = false;
  GlibcRandHost rng;
  HostSamples hs;
  // the device replay: pinned raw draws with the unread tail of the previous epoch in front, their device copy, the jump
  // tables, the consumed-draw counter
  int* h_raw = nullptr;
  long long raw_cap = 0, raw_have = 0, tables_cap = 0;
  DevBuf<int> d_raw, d_tables, d_consumed;
  void glibc_device_samples(long long n, cudaStream_t st);
};

}  // namespace b200
