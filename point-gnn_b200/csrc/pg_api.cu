// Library-wide C-ABI plumbing: version, error string, device probe, launch counter.
#include <atomic>
#include <stdarg.h>
#include <string.h>

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
