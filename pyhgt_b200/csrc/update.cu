// HGTConv.update epilogue (conv.py:129-133): sigmoid(skip)-gated residual + per-type LayerNorm.
// One warp per node row; the row (d <= 1024 floats) stays in registers between the two LayerNorm passes.
// HBM-bound: reads o and x (2*d*4 B), writes out (d*4 B) per node.
// DROP instances (hgt_update_epilogue_drop) scale `o` by a counter-based dropout mask as the row is loaded; the mask is a
// function of (seed, row, column) alone (hgt_b200.h, "Fused dropout"), so nothing is stored for the backward.
// hgt_tanh_dropout[_bwd] is the same mask behind the GNN adapter's tanh.
#include <cuda_bf16.h>

#include "common.cuh"

namespace {

constexpr int kMaxPerLane = 32;   // d <= 1024

template <bool DROP>
__global__ void __launch_bounds__(256)
k_update_epilogue(const float* __restrict__ o, const float* __restrict__ x, const int32_t* __restrict__ type_row0,
                  int T, const float* __restrict__ skip, const float* __restrict__ norm_w,
                  const float* __restrict__ norm_b, const float* const* __restrict__ norm_wp,
                  const float* const* __restrict__ norm_bp, const int32_t* __restrict__ perm,
                  const int32_t* __restrict__ type_active, const int32_t* __restrict__ type_dst,
                  const float* __restrict__ bias, int64_t n_nodes, int d, float* __restrict__ out,
                  const uint64_t* __restrict__ seed, uint32_t thr, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (row >= n_nodes) return;
  // node type of this rank: types are contiguous in rank order, T is small
  int t = 0;
  while (t < T && row >= type_row0[t + 1]) ++t;
  if (type_active && t < T && row - type_row0[t] >= type_active[t]) return;   // halo source: no output row
  if (perm && perm[row] < 0) return;             // sharded out_map: -1 = row without an output (e.g. unknown-type halo)
  float* orow = out + (perm ? (int64_t)perm[row] : row) * d;
  if (t >= T) {                                  // type outside [0,T): the reference leaves zeros (conv.py:120)
    for (int c = lane; c < d; c += 32) orow[c] = 0.f;
    return;
  }
  // skip == NULL: plain residual y = o + x (DenseHGTConv, conv.py:261,273)
  const float alpha = skip ? 1.0f / (1.0f + __expf(-skip[t])) : 1.0f;    // torch.sigmoid(self.skip[t]), conv.py:129
  const float beta = skip ? 1.0f - alpha : 1.0f;
  // rows past type_dst[t] have no in-edges: their a_linear output is exactly the bias, and their `o` row was not written
  const float* op = (type_dst && row - type_row0[t] >= type_dst[t]) ? bias + (int64_t)t * d : o + row * d;
  const float* xp = x + row * d;
  uint32_t kept = 0;
  if constexpr (DROP) kept = hgt_drop_row_bits<kMaxPerLane>(hgt_drop_key(seed), row, d, thr, lane);
  float y[kMaxPerLane];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxPerLane; ++i) {
    int c = lane + i * 32;
    if (c < d) {
      float ov = op[c];
      if constexpr (DROP) ov = hgt_drop_apply(ov, (kept >> i) & 1u, scale);
      y[i] = ov * alpha + xp[c] * beta;                    // conv.py:131,133
      sum += y[i];
    } else {
      y[i] = 0.f;
    }
  }
  if (norm_w == nullptr && norm_wp == nullptr) {
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
      int c = lane + i * 32;
      if (c < d) orow[c] = y[i];
    }
    return;
  }
  for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  const float mean = sum / d;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxPerLane; ++i) {
    int c = lane + i * 32;
    if (c < d) {
      float dlt = y[i] - mean;
      var = fmaf(dlt, dlt, var);
    }
  }
  for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
  const float rstd = rsqrtf(var / d + 1e-5f);              // nn.LayerNorm eps (conv.py:40)
  const float* w = norm_wp ? norm_wp[t] : norm_w + (int64_t)t * d;
  const float* b = norm_bp ? norm_bp[t] : norm_b + (int64_t)t * d;
#pragma unroll
  for (int i = 0; i < kMaxPerLane; ++i) {
    int c = lane + i * 32;
    if (c < d) orow[c] = (y[i] - mean) * rstd * w[c] + b[c];
  }
}

// The next layer's projection GEMM consumes its input as a bf16 hi/lo split: emit it here instead of re-reading `out`.
__device__ __forceinline__ void split_store(uint2* hi, uint2* lo, int64_t idx, const float4& v) {
  const float f[4] = {v.x, v.y, v.z, v.w};
  __nv_bfloat16 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = __float2bfloat16_rn(f[j]);
    l[j] = __float2bfloat16_rn(f[j] - __bfloat162float(h[j]));
  }
  hi[idx] = *reinterpret_cast<uint2*>(h);
  if (lo) lo[idx] = *reinterpret_cast<uint2*>(l);            // NULL: hi only
}

// Vectorised variant: d % 4 == 0, each lane owns NV float4 chunks (chunk c = lane + 32*i), 128-bit loads/stores.
template <int NV, bool DROP>
__global__ void __launch_bounds__(256)
k_update_epilogue_vec(const float* __restrict__ o, const float* __restrict__ x, const int32_t* __restrict__ type_row0,
                      int T, const float* __restrict__ skip, const float* __restrict__ norm_w,
                      const float* __restrict__ norm_b, const float* const* __restrict__ norm_wp,
                      const float* const* __restrict__ norm_bp, const int32_t* __restrict__ perm,
                      const int32_t* __restrict__ type_active, const int32_t* __restrict__ type_dst,
                      const float* __restrict__ bias, int64_t n_nodes, int d, float* __restrict__ out,
                      uint2* __restrict__ out_hi, uint2* __restrict__ out_lo, const uint64_t* __restrict__ seed,
                      uint32_t thr, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (row >= n_nodes) return;
  const int nvec = d >> 2;
  if (type_active) {
    // sharded runs: most local rows may be halo sources without an output row — leave before touching their data
    int t0 = 0;
    while (t0 < T && row >= type_row0[t0 + 1]) ++t0;
    if (t0 < T && row - type_row0[t0] >= type_active[t0]) return;
    if (perm && perm[row] < 0) return;
  }
  const float4* op = reinterpret_cast<const float4*>(o + row * d);
  bool tail = false;
  if (type_dst) {
    // rows past type_dst[t] have no in-edges: their a_linear output is exactly the bias, and their `o` row was not written
    int t0 = 0;
    while (t0 < T && row >= type_row0[t0 + 1]) ++t0;
    if (t0 < T && row - type_row0[t0] >= type_dst[t0]) {
      tail = true;
      op = reinterpret_cast<const float4*>(bias + (int64_t)t0 * d);
    }
  }
  // issue the row loads first; the (short, warp-uniform) type search overlaps with them
  float4 ov[NV], xv[NV];
  const float4* xp = reinterpret_cast<const float4*>(x + row * d);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < nvec) { ov[i] = tail ? __ldg(op + c) : __ldcs(op + c); xv[i] = __ldcs(xp + c); }
    else { ov[i] = make_float4(0.f, 0.f, 0.f, 0.f); xv[i] = ov[i]; }
  }
  int t = 0;
  while (t < T && row >= type_row0[t + 1]) ++t;
  if (type_active && t < T && row - type_row0[t] >= type_active[t]) return;
  if (perm && perm[row] < 0) return;             // sharded out_map: -1 = row without an output
  float4* orow = reinterpret_cast<float4*>(out + (perm ? (int64_t)perm[row] : row) * d);
  if (t >= T) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        orow[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (out_hi) split_store(out_hi, out_lo, row * nvec + c, make_float4(0.f, 0.f, 0.f, 0.f));
      }
    }
    return;
  }
  const float alpha = skip ? 1.0f / (1.0f + __expf(-skip[t])) : 1.0f;
  const float beta = skip ? 1.0f - alpha : 1.0f;
  if constexpr (DROP) {                          // rows that left above drew nothing
    const uint2 key = hgt_drop_key(seed);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        const uint32_t kept = hgt_drop_keep4(key, (uint64_t)row * nvec + c, thr);
        ov[i].x = hgt_drop_apply(ov[i].x, kept & 1u, scale);
        ov[i].y = hgt_drop_apply(ov[i].y, kept & 2u, scale);
        ov[i].z = hgt_drop_apply(ov[i].z, kept & 4u, scale);
        ov[i].w = hgt_drop_apply(ov[i].w, kept & 8u, scale);
      }
    }
  }
  float4 y[NV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    y[i].x = ov[i].x * alpha + xv[i].x * beta;
    y[i].y = ov[i].y * alpha + xv[i].y * beta;
    y[i].z = ov[i].z * alpha + xv[i].z * beta;
    y[i].w = ov[i].w * alpha + xv[i].w * beta;
    sum += (y[i].x + y[i].y) + (y[i].z + y[i].w);
  }
  if (norm_w == nullptr && norm_wp == nullptr) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < nvec) {
        __stcs(orow + c, y[i]);
        if (out_hi) split_store(out_hi, out_lo, row * nvec + c, y[i]);
      }
    }
    return;
  }
  for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  const float mean = sum / d;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < nvec) {
      float a = y[i].x - mean, b = y[i].y - mean, e = y[i].z - mean, f = y[i].w - mean;
      var += (a * a + b * b) + (e * e + f * f);
    }
  }
  for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
  const float rstd = rsqrtf(var / d + 1e-5f);
  const float* wf = norm_wp ? norm_wp[t] : norm_w + (int64_t)t * d;
  const float* bf = norm_bp ? norm_bp[t] : norm_b + (int64_t)t * d;
  // pointer-table entries are separate parameters, possibly views at any float offset into one flat buffer
  // (vector_to_parameters, FSDP): they take scalar loads unless both are 16-byte aligned (warp-uniform)
  const bool wb_vec = ((reinterpret_cast<uintptr_t>(wf) | reinterpret_cast<uintptr_t>(bf)) & 15) == 0;
  const float4* w = reinterpret_cast<const float4*>(wf);
  const float4* b = reinterpret_cast<const float4*>(bf);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < nvec) {
      float4 wv, bv;
      if (wb_vec) {
        wv = __ldg(w + c);
        bv = __ldg(b + c);
      } else {
        wv = make_float4(__ldg(wf + 4 * c), __ldg(wf + 4 * c + 1), __ldg(wf + 4 * c + 2), __ldg(wf + 4 * c + 3));
        bv = make_float4(__ldg(bf + 4 * c), __ldg(bf + 4 * c + 1), __ldg(bf + 4 * c + 2), __ldg(bf + 4 * c + 3));
      }
      float4 r;
      r.x = (y[i].x - mean) * rstd * wv.x + bv.x;
      r.y = (y[i].y - mean) * rstd * wv.y + bv.y;
      r.z = (y[i].z - mean) * rstd * wv.z + bv.z;
      r.w = (y[i].w - mean) * rstd * wv.w + bv.w;
      __stcs(orow + c, r);
      if (out_hi) split_store(out_hi, out_lo, row * nvec + c, r);
    }
  }
}

template <int NV, bool DROP>
void launch_vec(const float* o, const float* x, const int32_t* type_row0, int T, const float* skip,
                const float* norm_w, const float* norm_b, const float* const* norm_wp, const float* const* norm_bp,
                const int32_t* perm, const int32_t* type_active, const int32_t* type_dst, const float* bias,
                int64_t n_nodes, int d, float* out, uint2* out_hi, uint2* out_lo, const uint64_t* seed, HgtDrop dp,
                cudaStream_t st) {
  const int warps_per_block = 8;
  unsigned grid = (unsigned)((n_nodes + warps_per_block - 1) / warps_per_block);
  k_update_epilogue_vec<NV, DROP><<<grid, warps_per_block * 32, 0, st>>>(
      o, x, type_row0, T, skip, norm_w, norm_b, norm_wp, norm_bp, perm, type_active, type_dst, bias, n_nodes, d, out,
      out_hi, out_lo, seed, dp.thr, dp.scale);
}

}  // namespace

int hgt_update_epilogue_impl(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                             const float* skip, const float* norm_w, const float* norm_b, const float* const* norm_wp,
                             const float* const* norm_bp, const int32_t* perm, const int32_t* type_active,
                             const int32_t* type_dst, const float* bias, int64_t n_nodes, int32_t d, float* out,
                             void* out_hi, void* out_lo, const uint64_t* seed, float p, cudaStream_t st) {
  HGT_REQUIRE(seed == nullptr || (type_dst == nullptr && p > 0.f),
              "hgt_update_epilogue_drop: dropout needs p > 0 and excludes type_dst (an inference-only table)");
  HGT_REQUIRE(type_dst == nullptr || (bias != nullptr && type_active == nullptr),
              "hgt_update_epilogue: type_dst needs the a_linear bias and excludes type_active");
  HGT_REQUIRE(d >= 1 && d <= 32 * kMaxPerLane, "hgt_update_epilogue: d=%d unsupported (max %d)", d,
              32 * kMaxPerLane);
  HGT_REQUIRE((norm_w == nullptr) == (norm_b == nullptr) && (norm_wp == nullptr) == (norm_bp == nullptr),
              "hgt_update_epilogue: LayerNorm weight and bias must go together");
  if (n_nodes == 0) return 0;
  // pointer-table LayerNorm vectors (norm_wp / norm_bp) may sit at any float offset: the vector kernel tests them
  // row by row and loads misaligned ones as scalars, so only the [T,d] arrays norm_w / norm_b are checked here
  const bool aligned = (d % 4 == 0) && ((reinterpret_cast<uintptr_t>(o) | reinterpret_cast<uintptr_t>(x) |
                                        reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(norm_w) |
                                        reinterpret_cast<uintptr_t>(norm_b) |
                                        reinterpret_cast<uintptr_t>(bias)) % 16 == 0);
  HGT_REQUIRE(out_hi != nullptr || out_lo == nullptr, "hgt_update_epilogue: out_lo needs out_hi");
  HGT_REQUIRE(out_hi == nullptr || (aligned && d % 8 == 0 && perm == nullptr && type_active == nullptr),
              "hgt_update_epilogue: the split output needs d %% 8 == 0, 16-byte aligned buffers and identity row order");
  uint2* hi2 = reinterpret_cast<uint2*>(out_hi);
  uint2* lo2 = reinterpret_cast<uint2*>(out_lo);
  const HgtDrop dp = seed ? hgt_drop_params(p) : HgtDrop{0u, 1.f, 1.f};
  if (aligned && d <= 1024) {
    const int nv = (d / 4 + 31) / 32;
#define HGT_UE(NV)                                                                                                      \
  do {                                                                                                                  \
    if (seed) launch_vec<NV, true>(o, x, type_row0, num_types, skip, norm_w, norm_b, norm_wp, norm_bp, perm, type_active, \
                                   type_dst, bias, n_nodes, d, out, hi2, lo2, seed, dp, st);                             \
    else launch_vec<NV, false>(o, x, type_row0, num_types, skip, norm_w, norm_b, norm_wp, norm_bp, perm, type_active,    \
                               type_dst, bias, n_nodes, d, out, hi2, lo2, seed, dp, st);                                 \
  } while (0)
    if (nv <= 1) HGT_UE(1);
    else if (nv <= 2) HGT_UE(2);
    else if (nv <= 4) HGT_UE(4);
    else HGT_UE(8);
#undef HGT_UE
    HGT_LAUNCH_CHECK();
    return 0;
  }
  const int warps_per_block = 8;
  unsigned grid = (unsigned)((n_nodes + warps_per_block - 1) / warps_per_block);
  if (seed)
    k_update_epilogue<true><<<grid, warps_per_block * 32, 0, st>>>(o, x, type_row0, num_types, skip, norm_w, norm_b,
                                                                   norm_wp, norm_bp, perm, type_active, type_dst, bias,
                                                                   n_nodes, d, out, seed, dp.thr, dp.scale);
  else
    k_update_epilogue<false><<<grid, warps_per_block * 32, 0, st>>>(o, x, type_row0, num_types, skip, norm_w, norm_b,
                                                                    norm_wp, norm_bp, perm, type_active, type_dst, bias,
                                                                    n_nodes, d, out, seed, dp.thr, dp.scale);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_update_epilogue(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                                   const float* skip, const float* norm_w, const float* norm_b,
                                   const int32_t* perm, const int32_t* type_active, int64_t n_nodes, int32_t d,
                                   float* out, void* out_hi, void* out_lo, void* stream_) {
  return hgt_update_epilogue_impl(o, x, type_row0, num_types, skip, norm_w, norm_b, nullptr, nullptr, perm,
                                  type_active, nullptr, nullptr, n_nodes, d, out, out_hi, out_lo, nullptr, 0.f,
                                  (cudaStream_t)stream_);
}

extern "C" int hgt_update_epilogue_dst(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                                       const float* skip, const float* norm_w, const float* norm_b, const int32_t* perm,
                                       const int32_t* type_dst, const float* bias, int64_t n_nodes, int32_t d,
                                       float* out, void* out_hi, void* out_lo, void* stream_) {
  HGT_REQUIRE(type_dst && bias, "hgt_update_epilogue_dst: NULL type_dst / bias");
  return hgt_update_epilogue_impl(o, x, type_row0, num_types, skip, norm_w, norm_b, nullptr, nullptr, perm, nullptr,
                                  type_dst, bias, n_nodes, d, out, out_hi, out_lo, nullptr, 0.f, (cudaStream_t)stream_);
}

extern "C" int hgt_update_epilogue_drop(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                                        const float* skip, const float* norm_w, const float* norm_b,
                                        const int32_t* perm, const int32_t* type_active, int64_t n_nodes, int32_t d,
                                        float* out, void* out_hi, void* out_lo, const uint64_t* seed, float p,
                                        void* stream_) {
  HGT_REQUIRE(seed, "hgt_update_epilogue_drop: NULL seed");
  return hgt_update_epilogue_impl(o, x, type_row0, num_types, skip, norm_w, norm_b, nullptr, nullptr, perm,
                                  type_active, nullptr, nullptr, n_nodes, d, out, out_hi, out_lo, seed, p,
                                  (cudaStream_t)stream_);
}

// ---- tanh + dropout of the GNN input adapter (model.py:75-76) -------------------------------------------------------------
namespace {

// One thread per 4-column chunk.  VEC: d % 4 == 0 and 16-byte aligned buffers (128-bit accesses); otherwise the chunk's
// columns go one by one (the last chunk of a row may be short).  BWD: x = dout, y = the forward's output, out = d x.
template <bool VEC, bool BWD>
__global__ void __launch_bounds__(256)
k_tanh_dropout(const float* x, const float* y, int64_t n_rows, int64_t n_total, int d, const uint64_t* __restrict__ seed,
               uint32_t thr, float scale, float keep, float* out) {
  const int nchunk = (d + 3) >> 2;
  const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (q >= n_total * nchunk) return;
  const int64_t row = q / nchunk;
  const int c = (int)(q - row * nchunk);
  const bool through = row >= n_rows;              // rows of unknown type pass unchanged
  const uint32_t kept = through ? 0u : hgt_drop_keep4(hgt_drop_key(seed), (uint64_t)q, thr);
  auto f = [&](float xv, float yv, uint32_t k) {
    if (through) return xv;
    if (!BWD) return hgt_drop_apply(tanhf(xv), k, scale);
    const float th = yv * keep;                    // kept: tanh(x) = out / scale
    return hgt_drop_apply(xv * (1.0f - th * th), k, scale);
  };
  if (VEC) {
    const float4 xv = __ldcs(reinterpret_cast<const float4*>(x) + q);
    float4 yv = xv;
    if (BWD) yv = __ldcs(reinterpret_cast<const float4*>(y) + q);
    float4 r;
    r.x = f(xv.x, yv.x, kept & 1u);
    r.y = f(xv.y, yv.y, kept & 2u);
    r.z = f(xv.z, yv.z, kept & 4u);
    r.w = f(xv.w, yv.w, kept & 8u);
    __stcs(reinterpret_cast<float4*>(out) + q, r);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = 4 * c + j;
      if (col < d) {
        const int64_t e = row * d + col;
        out[e] = f(x[e], BWD ? y[e] : 0.f, (kept >> j) & 1u);
      }
    }
  }
}

template <bool BWD>
int tanh_dropout_launch(const char* who, const float* x, const float* y, int64_t n_rows, int64_t n_total, int32_t d,
                        const uint64_t* seed, float p, float* out, cudaStream_t st) {
  HGT_REQUIRE(x && out && seed && (y || !BWD), "%s: NULL argument", who);
  HGT_REQUIRE(d >= 1 && n_rows >= 0 && n_rows <= n_total && p > 0.f, "%s: needs d >= 1, 0 <= n_rows <= n_total, p > 0", who);
  if (n_total == 0) return 0;
  const HgtDrop dp = hgt_drop_params(p);
  const int64_t n = n_total * ((d + 3) / 4);
  const unsigned grid = (unsigned)((n + 255) / 256);
  const bool vec = d % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
                                   reinterpret_cast<uintptr_t>(out)) % 16 == 0);
  if (vec) k_tanh_dropout<true, BWD><<<grid, 256, 0, st>>>(x, y, n_rows, n_total, d, seed, dp.thr, dp.scale, dp.keep, out);
  else k_tanh_dropout<false, BWD><<<grid, 256, 0, st>>>(x, y, n_rows, n_total, d, seed, dp.thr, dp.scale, dp.keep, out);
  HGT_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int hgt_tanh_dropout(const float* x, int64_t n_rows, int64_t n_total, int32_t d, const uint64_t* seed,
                                float p, float* out, void* stream_) {
  return tanh_dropout_launch<false>("hgt_tanh_dropout", x, nullptr, n_rows, n_total, d, seed, p, out,
                                    (cudaStream_t)stream_);
}

extern "C" int hgt_tanh_dropout_bwd(const float* dout, const float* out, int64_t n_rows, int64_t n_total, int32_t d,
                                    const uint64_t* seed, float p, float* d_x, void* stream_) {
  return tanh_dropout_launch<true>("hgt_tanh_dropout_bwd", dout, out, n_rows, n_total, d, seed, p, d_x,
                                   (cudaStream_t)stream_);
}
