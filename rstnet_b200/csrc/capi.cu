// Error reporting, version and launch accounting for the C ABI (include/rstnet_b200.h).
#include "common.cuh"
#include "../../include/rstnet_b200.h"
#include <atomic>
#include <cstdarg>

namespace rstnet {

static thread_local char g_err[512] = {0};
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// Launch-configuration errors only (cudaGetLastError does not synchronise, and is legal during
// stream capture); asynchronous faults surface at the caller's next synchronisation.
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return 2;
  }
  return 0;
}

}  // namespace rstnet

namespace rstnet {
unsigned int lm_read_errors(bool clear);
unsigned int rvq_read_errors(bool clear);
unsigned int ce_read_errors(bool clear);
}

extern "C" int rstnet_version(void) { return 206; }
// Sticky device-side error bits of the CURRENT device (synchronises it): 1 = token / code id outside its table,
// 2 = RoPE position beyond the cos/sin tables.  Kernels cannot raise; they poison their output (NaN) and set a bit.
extern "C" uint32_t rstnet_device_error_flags(int clear) {
  cudaDeviceSynchronize();
  return rstnet::lm_read_errors(clear != 0) | rstnet::rvq_read_errors(clear != 0) | rstnet::ce_read_errors(clear != 0);
}
extern "C" const char* rstnet_last_error(void) { return rstnet::g_err; }
extern "C" int64_t rstnet_launch_count(void) { return rstnet::g_launches.load(); }
