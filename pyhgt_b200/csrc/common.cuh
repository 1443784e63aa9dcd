// Shared helpers for libhgt_b200.so (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "hgt_b200.h"

#define HGT_SM_COUNT_FALLBACK 132

void hgt_set_error(const char* fmt, ...);
int hgt_sm_count();

#define HGT_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      hgt_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));   \
      return 2;                                                                                   \
    }                                                                                             \
  } while (0)

#define HGT_REQUIRE(cond, ...)                                                                    \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      hgt_set_error(__VA_ARGS__);                                                                 \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

extern unsigned long long g_hgt_launches;   // kernels launched by this library (bench.py reports it)
#define HGT_LAUNCH_CHECK()                  \
  do {                                      \
    ++g_hgt_launches;                       \
    HGT_CHECK_CUDA(cudaGetLastError());     \
  } while (0)

static inline size_t hgt_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

__device__ __forceinline__ float hgt_gelu_erf(float x) {
  // F.gelu default (exact erf form), conv.py:119
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
