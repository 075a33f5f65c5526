// K2b: AsymmetricSVD epochs (Koren 2008), sm_90a.
//
// Replaces MatrixFactorization/Cython/MatrixFactorization_Cython_Epoch.pyx:396-578 epochIteration_Cython_ASY_SVD_SGD
// (batch size 1, :399), with sampleMSE_Cython :881-938 and adaptive_gradient :838-876.  The model is two n_items x f
// tables: Y (the reference's USER_factors, :163-166) and X (ITEM_factors).  A sample (u, i, r) reads the Y rows of the whole
// profile of u (their sum / sqrt(len_u) stands in for the user), predicts r with the X row of i, and then updates EVERY Y row
// of the profile and the X row of i, each parameter with its own adaptive state.
//
// The recursion is strictly sequential (sample t+1 reads rows sample t wrote: two profiles of ~150 items out of 27 K share
// an item more often than not), so ONE CTA walks the replayed sample stream in order and spreads the len_u x f reads and
// read-modify-writes of a sample over its 32 warps.  Per-phase cycle counters showed that
// the scalar one-warp-per-row version was ISSUE-bound (150 warp instructions per 32-element row, 24 K per sample on four
// schedulers), not latency-bound -- so rows are padded to a multiple of four factors and handled as float4s, min(32, f/4)
// lanes per row and several rows per warp instruction.
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "adaptive.cuh"
#include "common.cuh"
#include "sampler.cuh"

namespace b200 {
namespace asy {

constexpr int THREADS = 1024;
constexpr int WARPS = THREADS / 32;
static_assert(WARPS == 32, "step (2) keeps one partial vector per lane");

struct Params {
  int n_users, n_items, f, use_bias, sgd_mode;
  int fp, lpr;  // row stride (f rounded up to 4; the padding stays 0) and lanes per row (power of two <= min(32, fp / 8))
  float lr, user_reg, item_reg, bias_reg, gamma, beta1, beta2;
  double b1_pow, b2_pow;
  const int* __restrict__ indptr;
  const int* __restrict__ indices;
  float *Y, *X, *bu, *bi, *mu;
  float *cY, *cX, *cbu, *cbi, *cmu;            // adagrad / rmsprop cache, or adam first moment
  float *m2Y, *m2X, *m2bu, *m2bi, *m2mu;       // adam second moment
  const int* su; const int* si; const float* sr;
  long long n_samples;
  double* pow_out;
  int prof;  // B200REC_ASY_PROF=1: thread 0 times the phases of every sample and prints the averages (development hook)
};

// pyx:838-876 on register copies of the state; c is the adagrad / rmsprop cache or adam's first moment, m2 adam's second moment
__device__ __forceinline__ float adapt(const Params& p, float g, float& c, float& m2, float inv1, float inv2) {
  if (p.sgd_mode == B200_ADAGRAD) {
    c += g * g;
    return g / (sqrtf(c) + 1e-8f);
  } else if (p.sgd_mode == B200_RMSPROP) {
    c = c * p.gamma + (1.f - p.gamma) * g * g;
    return g / (sqrtf(c) + 1e-8f);
  } else if (p.sgd_mode == B200_ADAM) {
    c = c * p.beta1 + (1.f - p.beta1) * g;
    m2 = m2 * p.beta2 + (1.f - p.beta2) * g * g;
    return (c * inv1) / (sqrtf(m2 * inv2) + 1e-8f);
  }
  return g;
}
// the same on state that lives in memory (nullptr in the modes that have none)
__device__ __forceinline__ float adapt_at(const Params& p, float g, float* c, float* m2, float inv1, float inv2) {
  float cv = c ? *c : 0.f, mv = m2 ? *m2 : 0.f;
  const float r = adapt(p, g, cv, mv, inv1, inv2);
  if (c) *c = cv;
  if (m2) *m2 = mv;
  return r;
}

__device__ __forceinline__ float4 f4add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4shfl_xor(float4 a, int off) {
  return make_float4(__shfl_xor_sync(0xffffffffu, a.x, off), __shfl_xor_sync(0xffffffffu, a.y, off),
                     __shfl_xor_sync(0xffffffffu, a.z, off), __shfl_xor_sync(0xffffffffu, a.w, off));
}
// one float4 of a Y row: gradient, adaptive step, new value (pyx:510-521); c / m2 are updated in place
__device__ __forceinline__ float4 step4(const Params& p, float err, float4 h, float4 w, float4& c, float4& m2, float inv1, float inv2) {
  float4 o;
  o.x = w.x + p.lr * adapt(p, err * h.x - p.user_reg * w.x, c.x, m2.x, inv1, inv2);
  o.y = w.y + p.lr * adapt(p, err * h.y - p.user_reg * w.y, c.y, m2.y, inv1, inv2);
  o.z = w.z + p.lr * adapt(p, err * h.z - p.user_reg * w.z, c.z, m2.z, inv1, inv2);
  o.w = w.w + p.lr * adapt(p, err * h.w - p.user_reg * w.w, c.w, m2.w, inv1, inv2);
  return o;
}

// One CTA, samples strictly in order.  A warp instruction covers 32 / lpr rows of the profile (lane = row slot * lpr + sub;
// lane `sub` owns the float4s sub, sub + lpr of a 2 * lpr-float4 column block; rows wider than that are walked block by block).
// Per sample: (1) every lane sums its float4s over its rows, the row slots of a warp are added by shuffles, one partial
// vector per warp goes to shared memory; (2) warp w adds the 32 partial vectors for the factors w, w + 32, ..., reads the X
// row of the item and reduces the prediction; (3) thread 0 forms the error and steps the biases; (4) the Y rows (just read:
// L1) and their adaptive state are updated float4 by float4; (5) the X row.  The next sample's (user, item, rating) and
// profile bounds are fetched while the current one runs; inside a sample the item id of the next step is requested before
// the current step's rows.
// dynamic shared memory: part[WARPS][fp] partial profile sums, acc[fp] the profile vector, hx[fp] the X row before its update
#define ASY_MARK(k) do { if (p.prof && tid == 0) { const long long t_ = clock64(); prof[k] += (unsigned long long)(t_ - tprev); tprev = t_; } } while (0)
__global__ void __launch_bounds__(THREADS) asysvd_sequential_kernel(const Params p) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float red[WARPS];
  __shared__ float s_err, s_inv1, s_inv2;
  __shared__ unsigned long long prof[8];
  const int f = p.f, fp = p.fp, nq4 = fp >> 2, lpr = p.lpr;
  float* part = sm;
  float* acc = sm + (size_t)WARPS * fp;
  float* hx = acc + fp;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = lane & (lpr - 1), rpw = 32 / lpr, myrow0 = warp * rpw + lane / lpr, NR = WARPS * rpw;
  double b1p = p.b1_pow, b2p = p.b2_pow;  // advanced by thread 0 only
  long long tprev = 0;
  if (tid < 8) prof[tid] = 0ull;
  if (tid == 0) { s_inv1 = 1.f; s_inv2 = 1.f; }
  // sample n in (u, i, r, s, e); sample n + 1 in (nu, ni, nr)
  int u = 0, i = 0, s = 0, e = 0, nu = 0, ni = 0;
  float r = 0.f, nr = 0.f;
  if (p.n_samples > 0) { u = p.su[0]; i = p.si[0]; r = p.sr[0]; s = p.indptr[u]; e = p.indptr[u + 1]; }
  if (p.n_samples > 1) { nu = p.su[1]; ni = p.si[1]; nr = p.sr[1]; }
  __syncthreads();
  if (p.prof && tid == 0) tprev = clock64();
  for (long long n = 0; n < p.n_samples; ++n) {
    int nnu = 0, nni = 0;
    float nnr = 0.f;
    if (n + 2 < p.n_samples) { nnu = p.su[n + 2]; nni = p.si[n + 2]; nnr = p.sr[n + 2]; }
    const int ns = p.indptr[nu], ne = p.indptr[nu + 1];  // nu arrived an iteration ago (user 0 past the end: harmless)
    float b_mu = 0.f, b_u = 0.f, b_i = 0.f;
    if (tid == 0 && p.use_bias) { b_mu = p.mu[0]; b_u = p.bu[u]; b_i = p.bi[i]; }  // in flight during the gather
    const int len = e - s;
    // (1) pyx:436-448: sum of the Y rows of the profile
    for (int qb = 0; qb < nq4; qb += 2 * lpr) {
      const int q0 = qb + sub, q1 = q0 + lpr;
      float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
      int id = myrow0 < len ? p.indices[s + myrow0] : -1;
      for (int r0 = 0; r0 < len; r0 += NR) {  // warp-uniform trip count
        const int rn = r0 + NR + myrow0;
        const int idn = rn < len ? p.indices[s + rn] : -1;
        if (id >= 0) {
          const float4* row = reinterpret_cast<const float4*>(p.Y + (size_t)id * fp);
          if (q0 < nq4) a0 = f4add(a0, row[q0]);
          if (q1 < nq4) a1 = f4add(a1, row[q1]);
        }
        id = idn;
      }
      for (int off = lpr; off < 32; off <<= 1) { a0 = f4add(a0, f4shfl_xor(a0, off)); a1 = f4add(a1, f4shfl_xor(a1, off)); }
      if (lane < lpr) {
        float4* pw = reinterpret_cast<float4*>(part + (size_t)warp * fp);
        if (q0 < nq4) pw[q0] = a0;
        if (q1 < nq4) pw[q1] = a1;
      }
    }
    ASY_MARK(0);
    __syncthreads();
    ASY_MARK(1);
    // (2) warp w owns the factors w, w + 32, ...: the 32 partial vectors sit one per lane
    const float inv_den = 1.f / sqrtf((float)len);  // pyx:451-455
    float dot = 0.f;
    for (int q = warp; q < fp; q += WARPS) {
      float a = part[(size_t)lane * fp + q];
      const float h = q < f ? p.X[(size_t)i * fp + q] : 0.f;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
      a *= inv_den;
      if (lane == 0) { acc[q] = a; hx[q] = h; }
      dot += a * h;  // pyx:463-464 (every lane holds the same value)
    }
    if (lane == 0) red[warp] = dot;
    ASY_MARK(2);
    __syncthreads();
    ASY_MARK(3);
    // (3)
    if (warp == 0) {
      float pred = red[lane];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) pred += __shfl_xor_sync(0xffffffffu, pred, off);
      if (lane == 0) {
        float inv1 = 1.f, inv2 = 1.f;
        if (p.sgd_mode == B200_ADAM) { inv1 = adam_correction(b1p); inv2 = adam_correction(b2p); s_inv1 = inv1; s_inv2 = inv2; }
        if (p.use_bias) pred += b_mu + b_u + b_i;  // pyx:458-461
        const float err = r - pred;  // pyx:468-471 with batch_size == 1
        s_err = err;
        if (p.use_bias) {  // pyx:476-502: global, then item and user bias, all from the same error
          const float gm = adapt_at(p, err - p.bias_reg * b_mu, p.cmu, p.m2mu, inv1, inv2);
          const float gi = adapt_at(p, err - p.bias_reg * b_i, p.cbi ? p.cbi + i : nullptr, p.m2bi ? p.m2bi + i : nullptr, inv1, inv2);
          const float gu = adapt_at(p, err - p.bias_reg * b_u, p.cbu ? p.cbu + u : nullptr, p.m2bu ? p.m2bu + u : nullptr, inv1, inv2);
          p.mu[0] = b_mu + p.lr * gm;
          p.bi[i] = b_i + p.lr * gi;
          p.bu[u] = b_u + p.lr * gu;
        }
        if (p.sgd_mode == B200_ADAM) { b1p *= (double)p.beta1; b2p *= (double)p.beta2; }  // per sample, pyx:544-547
      }
    }
    ASY_MARK(4);
    __syncthreads();
    ASY_MARK(5);
    const float err = s_err, inv1 = s_inv1, inv2 = s_inv2;
    // (4) pyx:505-521: every Y row of the profile (the rows are distinct items), H_i from before the X update
    for (int qb = 0; qb < nq4; qb += 2 * lpr) {
      const int q0 = qb + sub, q1 = q0 + lpr;
      const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 h0 = q0 < nq4 ? reinterpret_cast<const float4*>(hx)[q0] : zero;
      const float4 h1 = q1 < nq4 ? reinterpret_cast<const float4*>(hx)[q1] : zero;
      int id = myrow0 < len ? p.indices[s + myrow0] : -1;
      for (int r0 = 0; r0 < len; r0 += NR) {
        const int rn = r0 + NR + myrow0;
        const int idn = rn < len ? p.indices[s + rn] : -1;
        if (id >= 0) {
          const size_t base4 = (size_t)id * nq4;
          float4* yrow = reinterpret_cast<float4*>(p.Y) + base4;
          float4* crow = p.cY ? reinterpret_cast<float4*>(p.cY) + base4 : nullptr;
          float4* mrow = p.m2Y ? reinterpret_cast<float4*>(p.m2Y) + base4 : nullptr;
          if (q0 < nq4) {
            float4 c = crow ? crow[q0] : zero, m2 = mrow ? mrow[q0] : zero;
            yrow[q0] = step4(p, err, h0, yrow[q0], c, m2, inv1, inv2);
            if (crow) crow[q0] = c;
            if (mrow) mrow[q0] = m2;
          }
          if (q1 < nq4) {
            float4 c = crow ? crow[q1] : zero, m2 = mrow ? mrow[q1] : zero;
            yrow[q1] = step4(p, err, h1, yrow[q1], c, m2, inv1, inv2);
            if (crow) crow[q1] = c;
            if (mrow) mrow[q1] = m2;
          }
        }
        id = idn;
      }
    }
    // (5) pyx:524-539: the X row of the sampled item, with the profile vector from before the Y update
    for (int q = tid; q < f; q += THREADS) {
      const size_t c = (size_t)i * fp + q;
      float g = err * acc[q] - p.item_reg * hx[q];
      g = adapt_at(p, g, p.cX ? p.cX + c : nullptr, p.m2X ? p.m2X + c : nullptr, inv1, inv2);
      p.X[c] = hx[q] + p.lr * g;
    }
    u = nu; i = ni; r = nr; s = ns; e = ne;
    nu = nnu; ni = nni; nr = nnr;
    ASY_MARK(6);
    __syncthreads();
    ASY_MARK(7);
  }
  if (tid == 0) {
    p.pow_out[0] = b1p; p.pow_out[1] = b2p;
    if (p.prof)
      printf("asysvd phase cycles per sample: gather=%llu bar1=%llu reduce=%llu bar2=%llu thread0=%llu bar3=%llu update=%llu bar4=%llu\n",
             prof[0] / p.n_samples, prof[1] / p.n_samples, prof[2] / p.n_samples, prof[3] / p.n_samples, prof[4] / p.n_samples,
             prof[5] / p.n_samples, prof[6] / p.n_samples, prof[7] / p.n_samples);
  }
}

}  // namespace asy
}  // namespace b200

using namespace b200;
using namespace b200::asy;

struct b200_asysvd_s {
  Params p{};
  SampleStream ss;
  DevBuf<float> Y, X, bu, bi, mu;
  AdaptBuffers sY, sX, sbu, sbi, smu;  // their optimiser state
  DevBuf<double> pow_out;
  EpochTimer timer;
};

extern "C" {

int b200_asysvd_create(b200_asysvd_t* out, int64_t n_users, int64_t n_items, int64_t nnz, const int32_t* h_indptr,
                       const int32_t* h_indices, const float* h_data, int n_factors, double negative_interactions_quota,
                       float learning_rate, int use_bias, float user_reg, float item_reg, float bias_reg, int sgd_mode,
                       float gamma, float beta_1, float beta_2, const double* h_profile_factors, const double* h_item_factors,
                       int has_seed, uint32_t random_seed) {
  if (out) *out = nullptr;
  b200_asysvd_s* h = nullptr;
  int rc = guarded([&] {
    B200_REQUIRE(out && h_indptr && h_indices && h_data && h_profile_factors && h_item_factors, "b200_asysvd_create: NULL argument");
    B200_REQUIRE(n_users > 0 && n_items > 0 && nnz > 0 && nnz < (1ll << 31) - 1, "b200_asysvd_create: bad shape");
    B200_REQUIRE(n_factors > 0 && n_factors <= 1024, "b200_asysvd_create: n_factors must be in [1, 1024] (got %d)", n_factors);
    B200_REQUIRE(sgd_mode >= B200_SGD && sgd_mode <= B200_ADAM, "b200_asysvd_create: unknown sgd_mode %d", sgd_mode);
    h = new b200_asysvd_s();
    Params& p = h->p;
    const size_t f = (size_t)n_factors, fp = (f + 3) & ~(size_t)3, nf = (size_t)n_items * fp;
    p.fp = (int)fp;
    p.lpr = 1;
    while (p.lpr * 2 <= std::min<int>(32, std::max<int>(1, (int)(fp / 8)))) p.lpr *= 2;  // a lane owns two float4s of a row
    p.n_users = (int)n_users; p.n_items = (int)n_items; p.f = n_factors; p.use_bias = use_bias != 0; p.sgd_mode = sgd_mode;
    p.lr = learning_rate; p.user_reg = user_reg; p.item_reg = item_reg; p.bias_reg = bias_reg;
    p.gamma = gamma; p.beta1 = beta_1; p.beta2 = beta_2;
    p.b1_pow = beta_1; p.b2_pow = beta_2;  // pyx:220-221
    const size_t n_epoch = (size_t)nnz + 1;  // pyx:402: int(len(data) / batch_size) + 1 with batch_size == 1
    h->ss.init(n_users, n_items, nnz, h_indptr, h_indices, h_data, false, negative_interactions_quota, n_epoch, false, 0,
               has_seed ? random_seed : 1u, false);
    p.indptr = h->ss.indptr.get(); p.indices = h->ss.indices.get();
    p.su = h->ss.su.get(); p.si = h->ss.si.get(); p.sr = h->ss.sr.get();
    upload_f32(h->Y, h_profile_factors, (size_t)n_items, f, fp); p.Y = h->Y.get();
    upload_f32(h->X, h_item_factors, (size_t)n_items, f, fp); p.X = h->X.get();
    h->bu.alloc_zeroed((size_t)n_users); h->bi.alloc_zeroed((size_t)n_items); h->mu.alloc_zeroed(1);  // pyx:184-186
    p.bu = h->bu.get(); p.bi = h->bi.get(); p.mu = h->mu.get();
    AdaptState a;  // pyx:248-270
    a = h->sY.alloc(sgd_mode, nf); p.cY = a.s1; p.m2Y = a.s2;
    a = h->sX.alloc(sgd_mode, nf); p.cX = a.s1; p.m2X = a.s2;
    a = h->sbu.alloc(sgd_mode, (size_t)n_users); p.cbu = a.s1; p.m2bu = a.s2;
    a = h->sbi.alloc(sgd_mode, (size_t)n_items); p.cbi = a.s1; p.m2bi = a.s2;
    a = h->smu.alloc(sgd_mode, 1); p.cmu = a.s1; p.m2mu = a.s2;
    h->pow_out.alloc(2);
    p.pow_out = h->pow_out.get();
    *out = h;
  });
  if (rc != B200_OK && h) delete h;
  return rc;
}

int b200_asysvd_destroy(b200_asysvd_t h) {
  if (!h) return B200_OK;
  delete h;
  return B200_OK;
}

int b200_asysvd_epoch(b200_asysvd_t h, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_asysvd_epoch: NULL handle");
    cudaStream_t st = (cudaStream_t)stream;
    Params& p = h->p;
    const long long n = (long long)h->ss.h_indices.size() + 1;
    p.n_samples = n;
    p.prof = getenv("B200REC_ASY_PROF") != nullptr;
    h->ss.draw_glibc(n, st);
    h->timer.begin(st);
    const size_t smem = (size_t)(WARPS + 2) * (size_t)p.fp * sizeof(float);
    // per launch: the attribute belongs to the function, and handles with other factor counts share it
    B200_CUDA(cudaFuncSetAttribute(asysvd_sequential_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1024)));
    asysvd_sequential_kernel<<<1, THREADS, smem, st>>>(p);
    B200_CUDA(cudaGetLastError());
    count_launch();
    h->timer.end(st);
    if (p.sgd_mode == B200_ADAM) read_powers(h->pow_out.get(), p.b1_pow, p.b2_pow, st);
    else if (h->ss.host_vectors_in_flight()) B200_CUDA(cudaStreamSynchronize(st));
  });
}

int b200_asysvd_get_samples(b200_asysvd_t h, int32_t* u, int32_t* i, float* r) {
  return guarded([&] {
    B200_REQUIRE(h && u && i && r && h->ss.drawn > 0, "b200_asysvd_get_samples: NULL argument or no epoch run yet");
    h->ss.copy_out(u, i, nullptr, r);
  });
}

int b200_asysvd_get_factors(b200_asysvd_t h, double* profile_factors, double* item_factors, double* user_bias, double* item_bias,
                            double* global_bias) {
  return guarded([&] {
    B200_REQUIRE(h != nullptr, "b200_asysvd_get_factors: NULL handle");
    B200_CUDA(cudaDeviceSynchronize());
    download_f64(profile_factors, h->Y.get(), (size_t)h->p.n_items, (size_t)h->p.f, (size_t)h->p.fp);
    download_f64(item_factors, h->X.get(), (size_t)h->p.n_items, (size_t)h->p.f, (size_t)h->p.fp);
    download_f64(user_bias, h->bu.get(), (size_t)h->p.n_users, 1, 1);
    download_f64(item_bias, h->bi.get(), (size_t)h->p.n_items, 1, 1);
    download_f64(global_bias, h->mu.get(), 1, 1, 1);
  });
}

int b200_asysvd_last_epoch_ms(b200_asysvd_t h, float* ms) {
  return guarded([&] {
    B200_REQUIRE(h && ms && h->timer.timed, "b200_asysvd_last_epoch_ms: no epoch run yet");
    h->timer.elapsed(ms);
  });
}

}  // extern "C"
