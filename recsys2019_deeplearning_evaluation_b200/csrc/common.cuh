// Shared plumbing for libb200rec.so: error reporting across the C ABI, launch accounting, device buffers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <new>
#include <vector>

#include "b200rec.h"

namespace b200 {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

struct CudaFail {
  int code;
};

#define B200_CUDA(expr)                                                                                  \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      b200::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e));      \
      throw b200::CudaFail{_e == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA};                \
    }                                                                                                    \
  } while (0)

#define B200_REQUIRE(cond, ...)             \
  do {                                      \
    if (!(cond)) {                          \
      b200::set_error(__VA_ARGS__);         \
      throw b200::CudaFail{B200_E_INVALID}; \
    }                                       \
  } while (0)

// Wraps a C-ABI body: converts internal throws into return codes.
template <typename F>
inline int guarded(F&& f) {
  try {
    f();
    return B200_OK;
  } catch (const CudaFail& e) {
    return e.code;
  } catch (const std::bad_alloc&) {
    set_error("host allocation failed");
    return B200_E_NOMEM;
  } catch (...) {
    set_error("unexpected internal error");
    return B200_E_CUDA;
  }
}

// Owning device buffer (cudaMalloc/cudaFree); move-only.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  explicit DevBuf(size_t count) { alloc(count); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t count) {
    release();
    n = count;
    if (count) B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&p), count * sizeof(T)));
  }
  void alloc_zeroed(size_t count) {
    alloc(count);
    if (count) B200_CUDA(cudaMemset(p, 0, count * sizeof(T)));
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  T* get() const { return p; }
};

// Host fp64 rows of f values -> device fp32 rows of ld >= f values; columns f..ld are zero
inline void upload_f32(DevBuf<float>& dst, const double* src, size_t rows, size_t f, size_t ld) {
  std::vector<float> tmp(rows * ld, 0.f);
  for (size_t r = 0; r < rows; ++r)
    for (size_t k = 0; k < f; ++k) tmp[r * ld + k] = (float)src[r * f + k];
  dst.alloc(rows * ld);
  B200_CUDA(cudaMemcpy(dst.get(), tmp.data(), rows * ld * sizeof(float), cudaMemcpyHostToDevice));
}

// Device fp32 rows of ld values -> host fp64 rows of their first f values; nothing when either side is null
inline void download_f64(double* dst, const float* src, size_t rows, size_t f, size_t ld) {
  if (!dst || !src) return;
  std::vector<float> tmp(rows * ld);
  B200_CUDA(cudaMemcpy(tmp.data(), src, rows * ld * sizeof(float), cudaMemcpyDeviceToHost));
  for (size_t r = 0; r < rows; ++r)
    for (size_t k = 0; k < f; ++k) dst[r * f + k] = (double)tmp[r * ld + k];
}

// Device time of a handle's last call (an epoch, a kernel): events recorded around the work on the caller's stream
struct EpochTimer {
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool timed = false;  // end() has run
  EpochTimer() {
    B200_CUDA(cudaEventCreate(&ev0));
    B200_CUDA(cudaEventCreate(&ev1));
  }
  EpochTimer(const EpochTimer&) = delete;
  EpochTimer& operator=(const EpochTimer&) = delete;
  ~EpochTimer() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
  }
  void begin(cudaStream_t st) { B200_CUDA(cudaEventRecord(ev0, st)); }
  void end(cudaStream_t st) {
    B200_CUDA(cudaEventRecord(ev1, st));
    timed = true;
  }
  void elapsed(float* ms) const {  // waits for the end event
    B200_CUDA(cudaEventSynchronize(ev1));
    B200_CUDA(cudaEventElapsedTime(ms, ev0, ev1));
  }
};

inline int sm_count() {
  int dev = 0, n = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  return n;
}

inline unsigned div_up(long long a, long long b) { return static_cast<unsigned>((a + b - 1) / b); }

}  // namespace b200
