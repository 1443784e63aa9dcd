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

// ---- bs16 gather tables (format: include/hgt_b200.h, "bs16 gather tables") -----------------------------------------
// Element type tag of the block-scaled 16-bit table: a row of n elements is hgt_bs16_row_bytes(n) bytes in two planes
// (n int16 mantissas, then n / 16 bf16 scales), addressed through hgt_bs16_at.
struct hgt_bs16 {};

__host__ __device__ __forceinline__ int64_t hgt_bs16_row_bytes(int64_t n) { return (2 * n + n / 8 + 15) / 16 * 16; }

// fp32(1 / (1 + i / 128)), i < 128: the correctly rounded reciprocal of a bf16 significand (a constant expression,
// rounded by the compiler)
struct HgtBs16RcpTab {
  float v[128];
};
constexpr HgtBs16RcpTab hgt_bs16_rcp_tab() {
  HgtBs16RcpTab t{};
  for (int i = 0; i < 128; ++i) t.v[i] = 1.0f / (1.0f + (float)i / 128.0f);
  return t;
}
static __device__ const HgtBs16RcpTab kHgtBs16Rcp = hgt_bs16_rcp_tab();

// Scale of a 16-element block from the largest |x| as fp32 bits (amax = max of bits & 0x7fffffff): the bf16 bits of s,
// and r, the factor the elements are multiplied by before rounding (0 where the block stores no mantissas).  Branch-free
// so that the epilogues overlap the blocks' shuffles and loads: r = 1 / s is the significand's reciprocal from the
// table with s's exponent negated, exact scaling by a power of two while 1 / s stays normal (s in [2^-126, 2^114]).
__device__ __forceinline__ uint32_t hgt_bs16_scale(uint32_t amax, float& r) {
  const float t = __fmul_rn(__uint_as_float(amax), 3.0518509447574615e-05f);  // fp32(1 / 32767)
  const uint32_t sb = (__float_as_uint(t) + 0xffffu) >> 16;                 // rounded up to bf16
  const int e = (int)((sb >> 7) & 0xffu);
  float rr = __uint_as_float(__float_as_uint(__ldg(&kHgtBs16Rcp.v[sb & 0x7fu])) + ((uint32_t)(127 - e) << 23));
  rr = sb >= 0x7780u ? __fmul_rn(rr, 0.999969482421875f) : rr;             // s >= 2^112: keep m * s below 2^128
  const bool nonfinite = amax >= 0x7f800000u;                               // NaN or Inf in the block: NaN scale,
                                                                            // zero mantissas (hgt_bs16_pack)
  const bool tiny = sb < 0x80u;                                             // s below FLT_MIN: the block stores zero
  r = nonfinite || tiny ? 0.f : rr;
  return nonfinite ? 0x7fc0u : tiny ? 0u : sb;
}

// Mantissas of two elements of a block with scale bits sb as (m0 & 0xffff) | (m1 << 16), m = rint_even(fl(x * r)):
// adding 1.5 * 2^23 rounds the product to an integer and leaves it, two's complement, in the low bits of the sum
// (|x * r| <= 32767.5).  A NaN-scale block stores zero mantissas.
__device__ __forceinline__ uint32_t hgt_bs16_pack(float x0, float x1, float r, uint32_t sb) {
  const float y0 = __fadd_rn(__fmul_rn(x0, r), 12582912.f), y1 = __fadd_rn(__fmul_rn(x1, r), 12582912.f);
  return sb == 0x7fc0u ? 0u : __byte_perm(__float_as_uint(y0), __float_as_uint(y1), 0x5410);
}

// Largest |x| bits over the 16-element block that the four lanes of an aligned quad hold (`a`: this lane's part).
__device__ __forceinline__ uint32_t hgt_bs16_quad_amax(uint32_t a) {
  a = max(a, __shfl_xor_sync(0xffffffffu, a, 1));
  return max(a, __shfl_xor_sync(0xffffffffu, a, 2));
}
__device__ __forceinline__ uint32_t hgt_abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }

// Element (row, col) of a table whose rows hold ld logical elements, given its logical offset off = row * ld + col:
// the byte of its mantissa and of its block's scale (col % 16 == 0 for the scale to be the block's first).
struct hgt_bs16_at {
  unsigned char* m;
  unsigned char* s;
  __host__ __device__ __forceinline__ hgt_bs16_at(void* base, int64_t off, int64_t ld) {
    const int64_t row = off / ld, col = off - row * ld;
    unsigned char* r = static_cast<unsigned char*>(base) + row * hgt_bs16_row_bytes(ld);
    m = r + 2 * col;
    s = r + 2 * ld + 2 * (col / 16);
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
