// Library-wide state: error string, launch counter, device properties.
#include "prl_common.cuh"
#include <atomic>
#include <string.h>
#include <stdlib.h>

namespace prl {

static thread_local char g_err[1024] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

static int g_pdl = -1;
bool use_pdl() {
  if (g_pdl < 0) {
    const char* e = getenv("PRL_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl == 1;
}

int num_sms() {
  static int cached[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace prl

extern "C" {
int prl_set_pdl(int32_t on) { prl::g_pdl = on ? 1 : 0; return PRL_OK; }
const char* prl_last_error(void) { return prl::g_err; }
int prl_version(void) { return 100; }
uint64_t prl_launch_count(void) { return prl::g_launches.load(std::memory_order_relaxed); }
}
