// api.cu -- library-wide plumbing of the C ABI: version, thread-local error text, launch counter.
#include <atomic>
#include "common.cuh"

namespace tfrs {
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {};
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  int& c = cached[dev & 63];
  if (!c) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) c = n;
    else return 132;
  }
  return c;
}
}  // namespace tfrs

extern "C" int tfrs_version(void) { return TFRS_B200_VERSION; }
extern "C" const char* tfrs_last_error(void) { return tfrs::g_err; }
extern "C" int64_t tfrs_launch_count(void) { return tfrs::g_launches.load(); }
