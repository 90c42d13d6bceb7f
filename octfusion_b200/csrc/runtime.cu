// Error text, version and device queries of the C ABI.
#include "common.cuh"
#include <string.h>

namespace of {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!cached[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}
static unsigned long long g_launches = 0;
void add_launches(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }
}  // namespace of

extern "C" unsigned long long of_launch_count(void) { return __atomic_load_n(&of::g_launches, __ATOMIC_RELAXED); }
extern "C" const char* of_last_error(void) { return of::g_err; }
extern "C" int of_version(void) { return 7; }
extern "C" int of_abi_sizeof_gemm_args(void) { return (int)sizeof(of_gemm_args); }
extern "C" int of_abi_sizeof_octree_levels(void) { return (int)sizeof(of_octree_levels); }
extern "C" int of_num_sms(void) { return of::num_sms(); }
