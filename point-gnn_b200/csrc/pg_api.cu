// Library-wide C-ABI plumbing: version, error string, device probe, launch counter, the CUB scans and sort.
#include <atomic>
#include <stdarg.h>
#include <string.h>

#include <cub/cub.cuh>

#include "pg_common.cuh"

namespace pg {
static thread_local char g_error[1024] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int exclusive_sum(const int32_t* in, int32_t* out, int64_t n, cudaStream_t s) {
  size_t bytes = 0;
  PG_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, int(n), s));
  Temp tmp;
  PG_CUDA_OK(tmp.alloc(bytes, s));
  PG_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp.ptr, bytes, in, out, int(n), s));
  count_launch(2);
  return PG_OK;
}

int inclusive_sum(const int32_t* in, int32_t* out, int64_t n, cudaStream_t s) {
  size_t bytes = 0;
  PG_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, in, out, int(n), s));
  Temp tmp;
  PG_CUDA_OK(tmp.alloc(bytes, s));
  PG_CUDA_OK(cub::DeviceScan::InclusiveSum(tmp.ptr, bytes, in, out, int(n), s));
  count_launch(2);
  return PG_OK;
}

int sort_pairs(const uint64_t* keys_in, uint64_t* keys_out, const int32_t* vals_in, int32_t* vals_out, int64_t n,
               int end_bit, cudaStream_t s) {
  size_t bytes = 0;
  PG_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys_in, keys_out, vals_in, vals_out, int(n), 0, end_bit, s));
  Temp tmp;
  PG_CUDA_OK(tmp.alloc(bytes, s));
  PG_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp.ptr, bytes, keys_in, keys_out, vals_in, vals_out, int(n), 0, end_bit, s));
  count_launch(4);
  return PG_OK;
}
}  // namespace pg

extern "C" {

int pg_version(void) { return 1; }

const char* pg_last_error(void) { return pg::g_error; }

int pg_device_is_sm90(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}

// the wgmma kernels are always built in, so the device decides
int pg_tc_available(void) { return pg_device_is_sm90(); }

int64_t pg_launch_count(void) { return pg::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
