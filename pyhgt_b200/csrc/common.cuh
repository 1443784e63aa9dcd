// Shared helpers for libhgt_b200.so (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <curand_philox4x32_x.h>   // curand_Philox4x32_10: the raw ten-round block function, no generator state
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

// ---- 24-bit gather tables (format: include/hgt_b200.h, "24-bit gather tables") -------------------------------------
// Element type tag of the planar 24-bit table: kernels templated on a table element type take it like float or bf16,
// but a row of n elements is 3n bytes in two planes, so it is addressed through hgt_t24_at, never by pointer arithmetic.
struct hgt_t24 {};

// fp32 word -> the rounded word whose bits 31..8 are stored (bits 7..0 are zero).
__host__ __device__ __forceinline__ uint32_t hgt_t24_round(uint32_t b) {
  const uint32_t r = (b + 0x7fu + ((b >> 8) & 1u)) & 0xffffff00u;   // past FLT_MAX the carry lands on Inf; Inf stays
  // NaN: quiet, sign kept (the add could carry a NaN into Inf or into the sign bit)
  return (b & 0x7fffffffu) > 0x7f800000u ? ((b | 0x00400000u) & 0xffffff00u) : r;
}

// Element (row, col) of a table whose rows hold ld logical elements, given its logical offset off = row * ld + col:
// the byte of its hi (u16) and of its lo (u8); element col + j has them 2 j and j bytes further.
struct hgt_t24_at {
  unsigned char* hi;
  unsigned char* lo;
  __host__ __device__ __forceinline__ hgt_t24_at(void* base, int64_t off, int64_t ld) {
    const int64_t row = off / ld, col = off - row * ld;
    hi = static_cast<unsigned char*>(base) + row * 3 * ld + 2 * col;
    lo = static_cast<unsigned char*>(base) + row * 3 * ld + 2 * ld + col;
  }
};

// ---- in-kernel dropout (mask contract: include/hgt_b200.h, "Fused dropout") ------------------------------------------
// Host side of the contract: keep threshold and scale of a drop probability p > 0.
struct HgtDrop {
  uint32_t thr;     // column kept iff its Philox word >= thr
  float scale;      // 1 / (1 - p); 0 for p >= 1 (everything dropped)
  float keep;       // 1 - p
};
static inline HgtDrop hgt_drop_params(float p) {
  HgtDrop r;
  if (p >= 1.0f) {
    r.thr = 0xffffffffu;
    r.scale = r.keep = 0.f;
  } else {
    r.thr = (uint32_t)((double)p * 4294967296.0);
    r.keep = 1.0f - p;
    r.scale = 1.0f / r.keep;
  }
  return r;
}

__device__ __forceinline__ uint2 hgt_drop_key(const uint64_t* __restrict__ seed) {
  const uint64_t s = *seed;
  return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

// Keep bits of the 4-column chunk q = row * ceil(d / 4) + col / 4: bit j belongs to column 4 * (col / 4) + j.
__device__ __forceinline__ uint32_t hgt_drop_keep4(uint2 key, uint64_t q, uint32_t thr) {
  const uint4 r = curand_Philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(q >> 32), 0u, 0u), key);
  return (uint32_t)(r.x >= thr) | ((uint32_t)(r.y >= thr) << 1) | ((uint32_t)(r.z >= thr) << 2) |
         ((uint32_t)(r.w >= thr) << 3);
}

// Keep bits of one row for the layout "lane owns columns lane + 32 * i, i < NPL" (NPL <= 32): bit i of the result.
// The four lanes of a quad share the chunk of column lane + 32 * i, so lane (quad base + j) draws the chunks of the
// i = j (mod 4) and the quad exchanges them: one Philox call per four columns.  Every lane of the warp must call it.
template <int NPL>
__device__ __forceinline__ uint32_t hgt_drop_row_bits(uint2 key, int64_t row, int d, uint32_t thr, int lane) {
  const int nchunk = (d + 3) >> 2;
  uint32_t bits = 0;
#pragma unroll
  for (int i0 = 0; i0 < NPL; i0 += 4) {
    const int chunk = (lane >> 2) + 8 * (i0 + (lane & 3));
    const uint32_t mine = chunk < nchunk ? hgt_drop_keep4(key, (uint64_t)row * nchunk + chunk, thr) : 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t theirs = __shfl_sync(0xffffffffu, mine, (lane & ~3) + j);
      if (i0 + j < NPL) bits |= ((theirs >> (lane & 3)) & 1u) << (i0 + j);
    }
  }
  return bits;
}

__device__ __forceinline__ float hgt_drop_apply(float v, uint32_t kept, float scale) { return kept ? v * scale : 0.f; }
