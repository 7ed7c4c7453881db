// Shared helpers for libpointgnn_b200 (error plumbing, launch accounting, temp buffers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <float.h>

#include "../../include/pointgnn_b200.h"

namespace pg {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// true while the current C-ABI call carries PG_FLAG_TRUSTED_INDICES (no range-error read-back, no sync)
bool trusted_indices();
void set_trusted_indices(bool v);

#define PG_CUDA_OK(expr)                                                              \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      pg::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return PG_ERR_CUDA;                                                             \
    }                                                                                 \
  } while (0)

#define PG_REQUIRE(cond, ...)              \
  do {                                     \
    if (!(cond)) {                         \
      pg::set_error(__VA_ARGS__);          \
      return PG_ERR_INVALID_ARGUMENT;      \
    }                                      \
  } while (0)

#define PG_LAUNCH_CHECK()                     \
  do {                                        \
    pg::count_launch();                       \
    PG_CUDA_OK(cudaGetLastError());           \
  } while (0)

// Stream-ordered temporary buffer; freed (stream-ordered) when it goes out of scope.
struct Temp {
  void* ptr = nullptr;
  cudaStream_t stream = nullptr;
  Temp() {}
  Temp(const Temp&) = delete;
  Temp& operator=(const Temp&) = delete;
  Temp(Temp&& o) noexcept : ptr(o.ptr), stream(o.stream) { o.ptr = nullptr; }
  cudaError_t alloc(size_t bytes, cudaStream_t s) {
    stream = s;
    if (bytes == 0) bytes = 16;
    keep_pool_warm();
    return cudaMallocAsync(&ptr, bytes, s);
  }
  // By default the stream-ordered pool returns freed memory to the OS at every synchronisation,
  // which turns each temporary into a driver allocation (measured: graph build 2.8 -> 26 ms/step).
  static void keep_pool_warm() {
    static bool done = false;
    if (done) return;
    done = true;
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long threshold = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
    }
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(ptr); }
  ~Temp() {
    if (ptr) cudaFreeAsync(ptr, stream);
  }
};

inline int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace pg
