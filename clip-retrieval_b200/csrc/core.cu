// Error plumbing and small process-wide state of the b200clip library.
#include "common.cuh"
#include <mutex>

namespace b200 {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count(int device) {
  static int cached[64];
  static std::once_flag once;
  std::call_once(once, [] { for (int& c : cached) c = 0; });
  if (device < 0 || device >= 64) return 132;
  if (cached[device] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    cached[device] = n;
  }
  return cached[device];
}

}  // namespace b200

extern "C" const char* b200_last_error(void) { return b200::g_err; }
extern "C" const char* b200_version(void) { return "b200clip 0.1 (sm_90a)"; }
extern "C" int64_t b200_launch_count(void) { return (int64_t)b200::g_launches.load(); }
