// Error channel + small utilities shared by every translation unit of libhgt_b200.so.
#include "common.cuh"

#include <string.h>

static thread_local char g_err[1024] = "";

void hgt_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int hgt_sm_count() {
  static int cached = 0;
  if (cached) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    n = HGT_SM_COUNT_FALLBACK;
  cached = n;
  return n;
}

unsigned long long g_hgt_launches = 0;

extern "C" uint64_t hgt_kernel_launches(void) { return g_hgt_launches; }
extern "C" const char* hgt_last_error(void) { return g_err; }
extern "C" int hgt_abi_version(void) { return 5; }
