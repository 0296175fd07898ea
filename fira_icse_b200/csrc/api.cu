// ABI bookkeeping: version, per-thread error string.
#include <stdarg.h>
#include "common.cuh"
#include "fira_b200.h"

#include <atomic>
#include <stdlib.h>

namespace {
thread_local char g_err[512] = "";
// launch mode (process-wide, atomic): -1 = not decided yet -> FIRA_PDL from the environment, default on
std::atomic<int> g_pdl{-1};
}

int fira_pdl_on() {
  int v = g_pdl.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("FIRA_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
    g_pdl.store(v, std::memory_order_relaxed);
  }
  return v;
}

void fira_set_error(int code, const char* fmt, ...) {
  int n = snprintf(g_err, sizeof(g_err), "[fira error %d] ", code);
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err + n, sizeof(g_err) - n, fmt, ap);
  va_end(ap);
}

extern "C" {
int fira_version(void) { return 3; }
const char* fira_last_error_string(void) { return g_err; }
int fira_built_arch(void) { return 90; }
int fira_num_sms(void) {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
  const int slot = dev < 64 ? dev : 63;
  int n = dev < 64 ? cache[slot].load(std::memory_order_relaxed) : 0;
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = 132;                                   // no device to ask: the H100 SXM
    }
    if (dev < 64) cache[slot].store(n, std::memory_order_relaxed);
  }
  return n;
}
int fira_set_pdl(int on) { g_pdl.store(on ? 1 : 0, std::memory_order_relaxed); return 0; }
int fira_get_pdl(void) { return fira_pdl_on(); }
}
