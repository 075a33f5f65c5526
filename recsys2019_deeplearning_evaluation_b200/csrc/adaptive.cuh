// The reference's optimiser step: adaptive_gradient (MatrixFactorization pyx:838-876) and Adam's bias corrections.
// The MF trainers (mf_sgd.cu) take the whole step from here; SLIM-BPR and AsySVD take the modes (b200_sgd_mode's), the
// bias correction and the host's bookkeeping of the Adam powers.  Every expression keeps the reference's operand order:
// fp32 contraction into FMAs depends on it, and the parity tests compare with the reference's arithmetic.
#pragma once
#include <math.h>

#include "common.cuh"

namespace b200 {

struct AdaptRule {
  int mode;  // b200_sgd_mode
  float gamma, beta1, beta2;
  float inv1, inv2;  // this step's Adam bias corrections, adam_correction(beta^t)
};

// 1 / (1 - beta^t) from the power beta^t
__host__ __device__ __forceinline__ float adam_correction(double pw) { return (float)(1.0 / (1.0 - pw)); }

// pyx:838-876 on register copies of one element's state: s1 is the adagrad / rmsprop cache or Adam's first moment, s2
// Adam's second moment
__device__ __forceinline__ float adapt(const AdaptRule& a, float g, float& s1, float& s2) {
  if (a.mode == B200_ADAGRAD) {
    s1 = s1 + g * g;
    return g / (sqrtf(s1) + 1e-8f);
  } else if (a.mode == B200_RMSPROP) {
    s1 = s1 * a.gamma + (1.f - a.gamma) * g * g;
    return g / (sqrtf(s1) + 1e-8f);
  } else if (a.mode == B200_ADAM) {
    s1 = s1 * a.beta1 + (1.f - a.beta1) * g;
    s2 = s2 * a.beta2 + (1.f - a.beta2) * g * g;
    return (s1 * a.inv1) / (sqrtf(s2 * a.inv2) + 1e-8f);
  }
  return g;
}

// How the pointer form reaches the state in memory
struct PlainAccess {  // ordinary loads and stores
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
struct L2Access {  // L2 only: rows stepped by other SMs leave no stale L1 line (mf_dataflow_kernel)
  static __device__ __forceinline__ float ld(const float* p) { return __ldcg(p); }
  static __device__ __forceinline__ void st(float* p, float v) { __stcg(p, v); }
};

// The state arrays of one parameter table: s1 in every adaptive mode, s2 in Adam only; null where the mode has none
struct AdaptState {
  float *s1, *s2;
};

// Owns the zeroed state arrays of one parameter table of n elements
struct AdaptBuffers {
  DevBuf<float> s1, s2;
  AdaptState alloc(int mode, size_t n) {
    if (mode != B200_SGD) s1.alloc_zeroed(n);
    if (mode == B200_ADAM) s2.alloc_zeroed(n);
    return {s1.get(), s2.get()};
  }
};

// pyx:838-876 on element o of a table whose state is in memory: loads what the mode reads, stores it back.  An array is
// indexed only in the modes that have it.
template <class Access = PlainAccess>
__device__ __forceinline__ float adapt_at(const AdaptRule& a, float g, const AdaptState& s, size_t o) {
  if (a.mode == B200_ADAGRAD || a.mode == B200_RMSPROP) {
    float v1 = Access::ld(s.s1 + o), v2 = 0.f;
    const float r = adapt(a, g, v1, v2);
    Access::st(s.s1 + o, v1);
    return r;
  } else if (a.mode == B200_ADAM) {
    float v1 = Access::ld(s.s1 + o), v2 = Access::ld(s.s2 + o);
    const float r = adapt(a, g, v1, v2);
    Access::st(s.s1 + o, v1);
    Access::st(s.s2 + o, v2);
    return r;
  }
  return g;
}

// Adam's powers after n more steps (a kernel that takes n steps without reporting its powers back)
inline void advance_powers(float beta1, float beta2, double& b1_pow, double& b2_pow, double n) {
  b1_pow *= pow((double)beta1, n);
  b2_pow *= pow((double)beta2, n);
}

// Adam's powers as a kernel left them in d_pow[2]; synchronises the stream
inline void read_powers(const double* d_pow, double& b1_pow, double& b2_pow, cudaStream_t st) {
  double pw[2];
  B200_CUDA(cudaMemcpyAsync(pw, d_pow, sizeof(pw), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  b1_pow = pw[0];
  b2_pow = pw[1];
}

}  // namespace b200
