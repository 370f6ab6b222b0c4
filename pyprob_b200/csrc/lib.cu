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

// read at every launch (a getenv per eager launch; graph replays do not come here) so that tests can flip it in-process.
// PPB_PDL = 0: off; 1 (default): tensor-core kernels and the element-wise kernels between them (cell, pack, NLL); 2: also the
// observe-MLP backward kernels; 3: also Adam (early-resident blocks of levels 2 and 3 take SMs from the side-stream branches)
int ppb_pdl_level() {
  const char* e = getenv("PPB_PDL");
  return (e && e[0] >= '0' && e[0] <= '9') ? e[0] - '0' : 1;
}
bool ppb_pdl_enabled() { return ppb_pdl_level() > 0; }

extern "C" {

const char* ppb_last_error(void) { return g_err; }

int ppb_version(void) { return 100; }

int64_t ppb_launch_count(void) { return (int64_t)g_ppb_launches; }

int ppb_device_arch(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return -1;
  return p.major * 10 + p.minor;
}

}  // extern "C"
