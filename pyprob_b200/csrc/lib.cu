// Library-wide plumbing: thread-local error string, version, device probe.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";
unsigned long long g_ppb_launches = 0;

void ppb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Both switches are read at every call (a getenv per eager launch; graph replays do not come here) so that tests can flip
// them in-process.
// PPB_PDL=0 turns programmatic dependent launch off (plain stream order, the reference the PDL chains are tested against)
bool ppb_pdl_enabled() {
  const char* e = getenv("PPB_PDL");
  return !(e && e[0] == '0');
}
// PPB_PERSISTENT=0 launches the grouped tensor-core GEMM with one CTA per tile even when a phase has more tiles than SMs
bool ppb_persistent_enabled() {
  const char* e = getenv("PPB_PERSISTENT");
  return !(e && e[0] == '0');
}

extern "C" {

const char* ppb_last_error(void) { return g_err; }

int ppb_version(void) { return 102; }

int64_t ppb_launch_count(void) { return (int64_t)g_ppb_launches; }

int ppb_device_arch(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return -1;
  return p.major * 10 + p.minor;
}

}  // extern "C"
