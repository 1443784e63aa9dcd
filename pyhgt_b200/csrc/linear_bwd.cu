// Backward of the typed (per-node-type) linear layers — hgt_typed_linear_bwd.
//
// Forward (linear.cu / linear_tc.cu):  out[cblock c of group g][m, n] = sum_k A[a_row0_g + m, k] * W[w_row0_g + c*width + n, k] + b
// Backward, for the same group / column-block tables:
//   dA[a_row0_g + m, k]            = sum_c sum_n dOut_c[m, n] * W[w_row0_g + c*width + n, k]      ("dX":  K = n_cblocks * width)
//   dW[w_row0_g + c*width + n, k] += sum_m dOut_c[m, n] * A[a_row0_g + m, k]                      ("dW":  K = rows of the group)
//   db[w_row0_g + c*width + n]    += sum_m dOut_c[m, n]
// The reference gets these from autograd over per-edge nn.Linear calls (conv.py:96-104,125; OAG/train_paper_field.py:249).
//
// Tensor-core path (Hopper wgmma, tcp::split3_tile in tc_ptx.cuh): the same split-bf16 x3 scheme as the forward (x = hi + lo,
// three bf16 products in one fp32 register accumulator):
//   k_act_split / k_split_colsum   fp32 -> bf16 hi/lo (optionally gelu first); the dOut split pass also produces db
//   k_lin_dx_tc (DxJob)   128 x tile_n tiles of dA (persistent CTAs); K runs over (column block, 64-wide k-block); A operand = dOut tiles
//           (K-major), B operand = W^T (a transposed, zero-padded bf16 split of the small weight matrix);
//           epilogue: optional `+= dA`, optional `* gelu'(aux)` (the gelu in front of the a_linears, conv.py:119)
//   k_lin_dw_tc (DwJob)   dW tiles [128 of width] x [tile_n of K_in] (persistent CTAs), each a reduction over a chunk of the group's rows; both operands
//           are MN-major (the reduction index is the row index): TMA boxes {64 columns, 64 rows}, SWIZZLE_128B;
//           partial tiles are added with red.global.add.v2.f32
// Every (group, column block) gets its own tensor map (tight row extents => rows past the group are zero-filled by TMA, so the
// reduction never sees a neighbour's rows); the maps live in the workspace (global memory).
// SIMT fp32 path for shapes the tensor cores cannot take (width % 8, K % 16, overlapping groups such as the RTE tables).
// impl 3: the tensor-core kernels with one bf16 product (tcp P = 1, torch's "medium" float32 matmul precision): only the
// hi halves of dOut, A and W^T are written and read; db is still summed from the fp32 dOut.
// bf16 A (hgt_typed_linear_bwd_bf16a, dW and db only): A is the dW product's B operand as it is, exact in bf16 with a zero
// lo half, so the tensor cores run dOut_hi*A + dOut_lo*A (tcp P = 4; dOut_hi*A at impl 3) and the SIMT kernel widens A as
// it loads it.  Either way dW and db are bitwise those of the fp32 call on the widened A.
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

using namespace tcp;

// Tensor maps are read from global memory (written by k_upload earlier on the stream): acquire them for the TMA proxy.
__device__ __forceinline__ void map_acquire(const CUtensorMap* m) {
  asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(m) : "memory");
}

// Host tables (task table, group offsets, tensor maps) reach the workspace by value in k_upload's parameter block, not
// through a host-memory copy: a CUDA graph records kernel parameters when the launch is captured, so the backward can be
// captured and replayed with no host buffer that has to outlive the call.  The block stays within the classic 4 KB
// parameter limit.
constexpr uint32_t kUploadBytes = 4096 - 16;
struct UploadChunk {
  unsigned char* dst;
  uint32_t n;
  alignas(16) unsigned char bytes[kUploadBytes];
};
static_assert(sizeof(UploadChunk) == 4096, "k_upload's parameter block must stay at 4 KB");

__global__ void __launch_bounds__(256) k_upload(const __grid_constant__ UploadChunk c) {
  for (uint32_t i = threadIdx.x; i < c.n; i += blockDim.x) c.dst[i] = c.bytes[i];
}

int upload_bytes(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  UploadChunk c{};
  for (size_t o = 0; o < bytes; o += kUploadBytes) {
    c.dst = static_cast<unsigned char*>(dst) + o;
    c.n = (uint32_t)std::min(bytes - o, (size_t)kUploadBytes);
    memcpy(c.bytes, static_cast<const unsigned char*>(src) + o, c.n);
    k_upload<<<1, 256, 0, st>>>(c);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

__device__ __forceinline__ float gelu_grad(float x) {
  // d/dx [0.5 x (1 + erf(x / sqrt 2))]
  return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * __expf(-0.5f * x * x);
}

// lo == NULL: hi only
__device__ __forceinline__ void split4(const float (&v)[4], uint2* hi, uint2* lo) {
  __nv_bfloat16 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = __float2bfloat16_rn(v[j]);
    l[j] = __float2bfloat16_rn(v[j] - __bfloat162float(h[j]));
  }
  *hi = *reinterpret_cast<uint2*>(h);
  if (lo) *lo = *reinterpret_cast<uint2*>(l);
}

// ---- fp32 [rows, K] (row stride ld) -> act(x) as fp32 and/or the bf16 hi/lo split [rows, Kp] (lo NULL: hi only) ------
__global__ void k_act_split(const float* __restrict__ in, int64_t ld, int64_t rows, int K, int Kp, int act,
                            float* __restrict__ out_f32, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int vec_per_row = Kp / 4;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= rows * vec_per_row) return;
  const int64_t r = i / vec_per_row;
  const int c = (int)(i - r * vec_per_row) * 4;
  float v[4];
  const float* src = in + r * ld + c;
  if (c + 3 < K && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
    const float4 t = *reinterpret_cast<const float4*>(src);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = (c + j < K) ? src[j] : 0.f;
  }
  if (act == 1) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = hgt_gelu_erf(v[j]);
  }
  if (out_f32) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c + j < K) out_f32[r * K + c + j] = v[j];
  }
  if (hi) split4(v, reinterpret_cast<uint2*>(hi + r * Kp + c), lo ? reinterpret_cast<uint2*>(lo + r * Kp + c) : nullptr);
}

// ---- W [w_rows, K] -> W^T split, block-padded:  WT[k, blk*wpad + n] = W[blk*width + n, k], zero for n >= width (lo NULL:
// hi only) ------------------------------------------------------------------------------------------------------------
__global__ void k_wt_split(const float* __restrict__ W, int64_t w_rows, int K, int width, int wpad, int64_t wt_cols,
                           __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * wt_cols) return;
  const int k = (int)(i / wt_cols);
  const int64_t col = i - (int64_t)k * wt_cols;
  const int64_t blk = col / wpad;
  const int n = (int)(col - blk * wpad);
  float v = 0.f;
  const int64_t wr = blk * width + n;
  if (n < width && wr < w_rows) v = W[wr * K + k];
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// ---- dOut split pass + bias gradient ---------------------------------------------------------------------------------
struct GcTask {            // one (group, column block)
  int64_t out_off, ld, rows, a_row0;
  int32_t w_row;           // first W row of this column block
  int32_t has_bias;
  int32_t first_unit;      // scheduling prefix (meaning depends on the kernel)
  int32_t n_chunks;
  int32_t map_dout;        // index of the dOut hi map (lo = +1)
  int32_t map_x;           // index of the group's A hi map (lo = +1)
  int32_t group, wt_col0;  // wt_col0: first column of this block inside W^T
};

// One CTA = one task x SPLIT_ROWS rows.  Thread (cx, ry): float4 column cx*4, rows ry, ry+RY, ...; column sums are reduced
// across ry in shared memory and added to db with one atomic per column and CTA.
constexpr int SPLIT_ROWS = 256;
// DET: the column sums of a CTA go to its own row of db_part [unit][width] (reduced in unit order by k_reduce_rows).
template <bool DET>
__device__ __forceinline__ void split_colsum(const float* __restrict__ dout, const GcTask* __restrict__ tasks, int n_tasks,
                                             int width, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                             float* __restrict__ db) {
  __shared__ float red[256 * 4];
  int unit = blockIdx.x, t = 0;
  while (t + 1 < n_tasks && unit >= tasks[t + 1].first_unit) ++t;
  const GcTask tk = tasks[t];
  const int64_t r0 = (int64_t)(unit - tk.first_unit) * SPLIT_ROWS;
  const int64_t r1 = min(tk.rows, r0 + SPLIT_ROWS);
  const int vecs = width / 4;                       // width % 4 == 0 on this path
  const int cxn = min(vecs, 256);                   // threads along columns
  const int ryn = 256 / cxn;
  const int cx = threadIdx.x % cxn, ry = threadIdx.x / cxn;
  for (int base = 0; base < vecs; base += cxn) {              // uniform trip count (barriers inside)
    const int c0 = base + cx;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    if (ry < ryn && c0 < vecs) {
      for (int64_t r = r0 + ry; r < r1; r += ryn) {
        const int64_t off = tk.out_off + r * tk.ld + c0 * 4;
        const float4 v4 = *reinterpret_cast<const float4*>(dout + off);
        const float v[4] = {v4.x, v4.y, v4.z, v4.w};
        split4(v, reinterpret_cast<uint2*>(hi + off), lo ? reinterpret_cast<uint2*>(lo + off) : nullptr);
#pragma unroll
        for (int j = 0; j < 4; ++j) s[j] += v[j];
      }
    }
    if (db && tk.has_bias) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red[threadIdx.x * 4 + j] = s[j];
      __syncthreads();
      if (ry == 0 && c0 < vecs) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a = 0.f;
          for (int y = 0; y < ryn; ++y) a += red[(y * cxn + cx) * 4 + j];
          if constexpr (DET) db[(int64_t)unit * width + c0 * 4 + j] = a;
          else atomicAdd(db + tk.w_row + c0 * 4 + j, a);
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(256)
k_split_colsum(const float* __restrict__ dout, const GcTask* __restrict__ tasks, int n_tasks, int width,
               __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, float* __restrict__ db) {
  split_colsum<false>(dout, tasks, n_tasks, width, hi, lo, db);
}
__global__ void __launch_bounds__(256)
k_split_colsum_det(const float* __restrict__ dout, const GcTask* __restrict__ tasks, int n_tasks, int width,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, float* __restrict__ db_part) {
  split_colsum<true>(dout, tasks, n_tasks, width, hi, lo, db_part);
}

// ---- dX: dA tile = sum over (column block, k-block) of dOut tile x W^T tile --------------------------------------------
// A operand = dOut of the group's column blocks (K-major, two 64-row boxes), B operand = W^T (K-major, tile_n-row box).
// Output columns past K_in (tile padding) and rows past the group are not stored.
struct DxJob {
  const CUtensorMap* maps;
  int map_wt;
  const GcTask* tasks;
  const int32_t* group_task0;
  const int64_t* first_tile;   // [n_groups + 1] first dA tile of every group (in the workspace: any number of groups)
  const hgt_lin_group* groups;
  int n_groups, K_in, width, n_tiles_n, tile_n;
  float* dA;
  int accumulate;
  const float* gelu_aux;

  struct Tile {
    int m0, n0, task0, kb_per_c, n_cblocks;
    int64_t rows, a_row0;
  };

  __device__ int decode(int tile, Tile& t) const {
    int g = 0;
    while (g + 1 < n_groups && tile >= first_tile[g + 1]) ++g;
    const hgt_lin_group grp = groups[g];
    const int local = (int)(tile - first_tile[g]);
    const int mt = local / n_tiles_n, nt = local - mt * n_tiles_n;
    t.m0 = mt * BM;
    t.n0 = nt * tile_n;
    t.task0 = group_task0[g];
    t.kb_per_c = (width + BK - 1) / BK;
    t.rows = grp.m - t.m0;
    t.a_row0 = grp.a_row0 + t.m0;
    t.n_cblocks = grp.n_cblocks;
    return grp.n_cblocks * t.kb_per_c;
  }
  __device__ void prefetch(const Tile& t) const {
    map_acquire(maps + map_wt);
    map_acquire(maps + map_wt + 1);
    for (int c = 0; c < t.n_cblocks; ++c) {
      map_acquire(maps + tasks[t.task0 + c].map_dout);
      map_acquire(maps + tasks[t.task0 + c].map_dout + 1);
    }
  }
  template <int BN, int KB, int P>
  __device__ void load(const Tile& t, int it, uint32_t sa, uint32_t bar) const {
    static_assert(KB == BK, "64-wide k-blocks");
    constexpr uint32_t B = b_offset<BK, P>();
    const int c = it / t.kb_per_c, kb = it - c * t.kb_per_c;
    const GcTask& tk = tasks[t.task0 + c];
    const CUtensorMap* m_hi = maps + tk.map_dout;
    const CUtensorMap* m_lo = m_hi + 1;
    tma_load_2d(sa, m_hi, kb * BK, t.m0, bar);
    tma_load_2d(sa + ATOM_BYTES, m_hi, kb * BK, t.m0 + 64, bar);
    tma_load_2d(sa + B, maps + map_wt, tk.wt_col0 + kb * BK, t.n0, bar);
    if constexpr (P == 3) {
      tma_load_2d(sa + A_BYTES, m_lo, kb * BK, t.m0, bar);
      tma_load_2d(sa + A_BYTES + ATOM_BYTES, m_lo, kb * BK, t.m0 + 64, bar);
      tma_load_2d(sa + B + BN * BK * 2, maps + map_wt + 1, tk.wt_col0 + kb * BK, t.n0, bar);
    }
  }
  template <int BN>
  __device__ void store(const Tile& t, const float* acc, float*, int c, int wq, int lane) const {
    const int64_t rows = t.rows - 64 * c;
    const int cols = K_in - t.n0;
    const int64_t row0 = (t.a_row0 + 64 * c) * K_in + t.n0;
    float* o = dA + row0;
    const float* x = gelu_aux ? gelu_aux + row0 : nullptr;
    const int ld = K_in;
    const bool acc_in = accumulate != 0;
    for_each_pair<BN>(acc, wq, lane, [&](int r, int col, float v0, float v1) {
      if (r < rows && col < cols) {
        const int64_t off = (int64_t)r * ld + col;
        if (x) {
          const float2 xv = *reinterpret_cast<const float2*>(x + off);
          v0 *= gelu_grad(xv.x);
          v1 *= gelu_grad(xv.y);
        }
        if (acc_in) {
          const float2 ov = *reinterpret_cast<const float2*>(o + off);
          v0 += ov.x;
          v1 += ov.y;
        }
        *reinterpret_cast<float2*>(o + off) = make_float2(v0, v1);
      }
    });
  }
};

// ---- dW: [128 rows of the column block] x [tile_n columns of K_in] += dOut_c^T A over a chunk of rows -----------------
// Both operands MN-major (the reduction index is the row index): TMA boxes {64 columns, 64 rows}; partial tiles are added
// with red.global.add.v2.f32.
struct DwJob {
  const CUtensorMap* maps;
  const GcTask* tasks;
  int n_tasks, K_in, width, m_tiles, n_tiles, chunk_rows, tile_n;
  float* dW;

  struct Tile {
    int mt, n0, map_dout, map_x, w_row;
    int64_t r0;
  };

  __device__ int decode(int unit, Tile& t) const {
    int i = 0;
    while (i + 1 < n_tasks && unit >= tasks[i + 1].first_unit) ++i;
    const GcTask tk = tasks[i];
    int local = unit - tk.first_unit;
    const int chunk = local / (m_tiles * n_tiles);
    local -= chunk * m_tiles * n_tiles;
    t.mt = local / n_tiles;
    t.n0 = (local - t.mt * n_tiles) * tile_n;
    t.map_dout = tk.map_dout;
    t.map_x = tk.map_x;
    t.w_row = tk.w_row;
    t.r0 = (int64_t)chunk * chunk_rows;
    const int64_t r1 = min(tk.rows, t.r0 + chunk_rows);
    return (int)((r1 - t.r0 + BK - 1) / BK);
  }
  __device__ void prefetch(const Tile& t) const {
    map_acquire(maps + t.map_dout);
    map_acquire(maps + t.map_dout + 1);
    map_acquire(maps + t.map_x);
    map_acquire(maps + t.map_x + 1);
  }
  template <int BN, int KB, int P>
  __device__ void load(const Tile& t, int it, uint32_t sa, uint32_t bar) const {
    static_assert(KB == BK, "64-row k-blocks");
    constexpr uint32_t B = b_offset<BK, P>();
    const int row = (int)(t.r0 + (int64_t)it * BK);
    const CUtensorMap* d_hi = maps + t.map_dout;
    const CUtensorMap* x_hi = maps + t.map_x;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      tma_load_2d(sa + j * ATOM_BYTES, d_hi, t.mt * BM + j * 64, row, bar);
      if constexpr (has_a_lo<P>()) tma_load_2d(sa + A_BYTES + j * ATOM_BYTES, d_hi + 1, t.mt * BM + j * 64, row, bar);
    }
#pragma unroll
    for (int j = 0; j < BN / 64; ++j) {
      tma_load_2d(sa + B + j * ATOM_BYTES, x_hi, t.n0 + j * 64, row, bar);
      if constexpr (has_b_lo<P>()) tma_load_2d(sa + B + BN * BK * 2 + j * ATOM_BYTES, x_hi + 1, t.n0 + j * 64, row, bar);
    }
  }
  template <int BN>
  __device__ void store(const Tile& t, const float* acc, float*, int c, int wq, int lane) const {
    const int rows = width - t.mt * BM - 64 * c;                   // rows of the dW tile = columns of the dOut block
    const int cols = K_in - t.n0;
    float* o = dW + ((int64_t)t.w_row + t.mt * BM + 64 * c) * K_in + t.n0;
    const int ld = K_in;
    for_each_pair<BN>(acc, wq, lane, [&](int r, int col, float v0, float v1) {
      if (r < rows && col < cols)
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(o + (int64_t)r * ld + col), "f"(v0), "f"(v1)
                     : "memory");
    });
  }
};

// Deterministic dW: every unit (task, chunk, tile) stores its partial tile into its own [width, K_in] slot
// (slot = unit / (m_tiles * n_tiles) = the task's first chunk slot + chunk); k_reduce_rows adds the slots in chunk order.
struct DwJobDet : DwJob {
  float* part;

  struct Tile : DwJob::Tile {
    int64_t slot;
  };

  __device__ int decode(int unit, Tile& t) const {
    t.slot = unit / (m_tiles * n_tiles);
    return DwJob::decode(unit, t);
  }
  template <int BN>
  __device__ void store(const Tile& t, const float* acc, float*, int c, int wq, int lane) const {
    const int rows = width - t.mt * BM - 64 * c;
    const int cols = K_in - t.n0;
    float* o = part + (t.slot * width + t.mt * BM + 64 * c) * K_in + t.n0;
    const int ld = K_in;
    for_each_pair<BN>(acc, wq, lane, [&](int r, int col, float v0, float v1) {
      if (r < rows && col < cols) *reinterpret_cast<float2*>(o + (int64_t)r * ld + col) = make_float2(v0, v1);
    });
  }
};

// out[wr, k] += sum over the tasks covering W row wr (task order), over their slots (chunk order) of
// part[slot, wr - w_row, k].  slot = first_unit / units_per_slot + chunk, n_chunks slots per task.  One thread per
// element: each W row has one owner however many tasks share it.  k_cols = 1 reduces the bias partials.
__global__ void k_reduce_rows(const float* __restrict__ part, const GcTask* __restrict__ tasks, int n_tasks, int width,
                              int k_cols, int64_t w_rows, int units_per_slot, int bias_only, float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= w_rows * k_cols) return;
  const int64_t wr = i / k_cols;
  const int k = (int)(i - wr * k_cols);
  float s = 0.f;
  bool any = false;
  for (int t = 0; t < n_tasks; ++t) {
    const GcTask& tk = tasks[t];
    if (wr < tk.w_row || wr >= tk.w_row + width || (bias_only && !tk.has_bias)) continue;
    any = true;
    const int64_t slot0 = tk.first_unit / units_per_slot;
    const int64_t n = wr - tk.w_row;
    for (int c = 0; c < tk.n_chunks; ++c) s += part[((slot0 + c) * width + n) * k_cols + k];
  }
  if (any) out[i] += s;
}

// ---- SIMT fp32 fallbacks ------------------------------------------------------------------------------------------------
// dA[a_row0 + m, k] (+)= sum_c sum_n dOut_c[m, n] * W[w_row + n, k].  One thread per (m, k); atomicAdd because groups may
// share A rows (the RTE tables: every <type, relation> pair projects the same 240-row table).
__global__ void k_lin_dx_simt(const float* __restrict__ dout, const float* __restrict__ W, const GcTask* __restrict__ tasks,
                              const int32_t* __restrict__ group_task0, const hgt_lin_group* __restrict__ groups,
                              int n_groups, const int64_t* __restrict__ group_first, int K_in, int width,
                              const float* __restrict__ gelu_aux, float* __restrict__ dA) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int g = 0;
  while (g + 1 < n_groups && i >= group_first[g + 1]) ++g;
  if (i >= group_first[n_groups]) return;
  const hgt_lin_group grp = groups[g];
  const int64_t li = i - group_first[g];
  const int64_t m = li / K_in;
  const int k = (int)(li - m * K_in);
  float acc = 0.f;
  for (int c = 0; c < grp.n_cblocks; ++c) {
    const GcTask tk = tasks[group_task0[g] + c];
    const float* drow = dout + tk.out_off + m * tk.ld;
    const float* wcol = W + (int64_t)tk.w_row * K_in + k;
    for (int n = 0; n < width; ++n) acc = fmaf(drow[n], wcol[(int64_t)n * K_in], acc);
  }
  const int64_t o = (grp.a_row0 + m) * K_in + k;
  if (gelu_aux) acc *= gelu_grad(gelu_aux[o]);
  atomicAdd(dA + o, acc);
}

// Deterministic dA: one thread per element of rows [0, a_rows); the groups that cover the row are added in group order.
__global__ void k_lin_dx_simt_det(const float* __restrict__ dout, const float* __restrict__ W,
                                  const GcTask* __restrict__ tasks, const int32_t* __restrict__ group_task0,
                                  const hgt_lin_group* __restrict__ groups, int n_groups, int64_t a_rows, int K_in,
                                  int width, const float* __restrict__ gelu_aux, int accumulate, float* __restrict__ dA) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= a_rows * K_in) return;
  const int64_t row = i / K_in;
  const int k = (int)(i - row * K_in);
  float acc = 0.f;
  bool any = false;
  for (int g = 0; g < n_groups; ++g) {
    const hgt_lin_group grp = groups[g];
    if (row < grp.a_row0 || row >= grp.a_row0 + grp.m) continue;
    any = true;
    const int64_t m = row - grp.a_row0;
    for (int c = 0; c < grp.n_cblocks; ++c) {
      const GcTask tk = tasks[group_task0[g] + c];
      const float* drow = dout + tk.out_off + m * tk.ld;
      const float* wcol = W + (int64_t)tk.w_row * K_in + k;
      for (int n = 0; n < width; ++n) acc = fmaf(drow[n], wcol[(int64_t)n * K_in], acc);
    }
  }
  if (any && gelu_aux) acc *= gelu_grad(gelu_aux[i]);
  dA[i] = accumulate ? dA[i] + acc : acc;
}

// dW[w_row + n, k] += sum_m dOut_c[m, n] * A[a_row0 + m, k];  db[w_row + n] += sum_m dOut_c[m, n].
// One CTA = one task x (32 n) x (32 k) x a chunk of rows; 256 threads, 4 outputs each.  dW == NULL (db only): one k tile,
// A (which may then be NULL) is not read.
constexpr int DW_SIMT_ROWS = 2048;
// DET: partial tiles / bias sums go to the unit's slot (unit / (n_tiles * k_tiles)) of dW = part [slot][width][K_in] and
// db = db_part [slot][width]; chunks of chunk_rows rows.
__device__ __forceinline__ float load_a(const float* p) { return *p; }
__device__ __forceinline__ float load_a(const __nv_bfloat16* p) { return __bfloat162float(*p); }   // exact

template <bool DET, class AT>
__device__ __forceinline__ void lin_dw_simt(const float* __restrict__ dout, const AT* __restrict__ A, int64_t lda,
                                            const GcTask* __restrict__ tasks, int n_tasks, int K_in, int width,
                                            int n_tiles, int k_tiles, int64_t chunk_rows, float* __restrict__ dW,
                                            float* __restrict__ db) {
  __shared__ float sd[32][33], sa[32][33];
  int unit = blockIdx.x, t = 0;
  while (t + 1 < n_tasks && unit >= tasks[t + 1].first_unit) ++t;
  const GcTask tk = tasks[t];
  int local = unit - tk.first_unit;
  const int chunk = local / (n_tiles * k_tiles);
  local -= chunk * n_tiles * k_tiles;
  const int ntile = local / k_tiles, ktile = local - ntile * k_tiles;
  const int n0 = ntile * 32, k0 = ktile * 32;
  const int64_t r0 = (int64_t)chunk * chunk_rows, r1 = min(tk.rows, r0 + chunk_rows);
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // ty: 0..7
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float bsum = 0.f;
  for (int64_t rb = r0; rb < r1; rb += 32) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int rr = ty + 8 * j;
      const int64_t r = rb + rr;
      float dv = 0.f, av = 0.f;
      if (r < r1) {
        if (n0 + tx < width) dv = dout[tk.out_off + r * tk.ld + n0 + tx];
        if (dW && k0 + tx < K_in) av = load_a(A + (tk.a_row0 + r) * lda + k0 + tx);
      }
      sd[rr][tx] = dv;
      sa[rr][tx] = av;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr) {
      const float a = sa[rr][tx];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(sd[rr][ty + 8 * j], a, acc[j]);
    }
    if (ktile == 0 && ty == 0) {
      for (int rr = 0; rr < 32; ++rr) bsum += sd[rr][tx];
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = n0 + ty + 8 * j;
    if (dW && n < width && k0 + tx < K_in) {
      if constexpr (DET) dW[((int64_t)(unit / (n_tiles * k_tiles)) * width + n) * K_in + k0 + tx] = acc[j];
      else atomicAdd(dW + ((int64_t)tk.w_row + n) * K_in + k0 + tx, acc[j]);
    }
  }
  if (db && tk.has_bias && ktile == 0 && ty == 0 && n0 + tx < width) {
    if constexpr (DET) db[(int64_t)(unit / (n_tiles * k_tiles)) * width + n0 + tx] = bsum;
    else atomicAdd(db + tk.w_row + n0 + tx, bsum);
  }
}
template <class AT>
__global__ void __launch_bounds__(256)
k_lin_dw_simt(const float* __restrict__ dout, const AT* __restrict__ A, int64_t lda, const GcTask* __restrict__ tasks,
              int n_tasks, int K_in, int width, int n_tiles, int k_tiles, float* __restrict__ dW, float* __restrict__ db) {
  lin_dw_simt<false>(dout, A, lda, tasks, n_tasks, K_in, width, n_tiles, k_tiles, DW_SIMT_ROWS, dW, db);
}
template <class AT>
__global__ void __launch_bounds__(256)
k_lin_dw_simt_det(const float* __restrict__ dout, const AT* __restrict__ A, int64_t lda,
                  const GcTask* __restrict__ tasks, int n_tasks, int K_in, int width, int n_tiles, int k_tiles,
                  int64_t chunk_rows, float* __restrict__ dw_part, float* __restrict__ db_part) {
  lin_dw_simt<true>(dout, A, lda, tasks, n_tasks, K_in, width, n_tiles, k_tiles, chunk_rows, dw_part, db_part);
}

// ---- host helpers ---------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2-D bf16 map over [rows, cols] with row stride `ld` elements, box {64 columns, box_rows}, SWIZZLE_128B, OOB -> 0.
int make_map2(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  HGT_REQUIRE(fn != nullptr, "hgt_typed_linear_bwd: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)(rows > 0 ? rows : 1)};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HGT_REQUIRE(r == CUDA_SUCCESS, "hgt_typed_linear_bwd: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld",
              (int)r, (long long)rows, (long long)cols, (long long)ld);
  return 0;
}

struct BwdLayout {
  bool tc, one;              // tensor cores; one bf16 product (impl 3): no lo halves
  int Kp, wpad;
  int64_t a_rows, w_rows, wt_cols;
  int n_tasks;
  int64_t dw_chunk;          // rows per dW reduction chunk (deterministic mode)
  size_t off_maps, off_tasks, off_gt0, off_gfirst, off_dhi, off_dlo, off_ahi, off_alo, off_wthi, off_wtlo, total;
  size_t off_part, off_dbp;  // deterministic mode: dW partial slots [slot][width][K], bias partials [unit][width]
};

// Rows per chunk of the tensor-core dW reduction: a few waves of CTAs over all (task, tile) pairs.
int64_t tc_dw_chunk(int64_t task_rows, int width, int K) {
  const int64_t m_tiles = (width + BM - 1) / BM, n_tiles = (K + pick_tile_n(K) - 1) / pick_tile_n(K);
  int64_t chunk = task_rows * m_tiles * n_tiles / (4 * (int64_t)hgt_sm_count());
  chunk = (chunk + BK - 1) / BK * BK;
  if (chunk < 1024) chunk = 1024;
  if (chunk > 32768) chunk = 32768;
  return chunk;
}

// The SIMT dW keeps at most ~256 partial slots in deterministic mode (plus one per task for rounding).
int64_t simt_det_chunk(int64_t task_rows) {
  int64_t chunk = (task_rows + 255) / 256;
  chunk = (chunk + 31) / 32 * 32;
  return chunk < DW_SIMT_ROWS ? DW_SIMT_ROWS : chunk;
}

bool groups_overlap(const hgt_lin_group* h, int n) {
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j) {
      if (h[i].m == 0 || h[j].m == 0) continue;
      if (h[i].a_row0 < h[j].a_row0 + h[j].m && h[j].a_row0 < h[i].a_row0 + h[i].m) return true;
    }
  return false;
}

bool bwd_tc_ok(const hgt_lin_group* h_groups, int n_groups, const hgt_lin_cblock* h_cb, int K, int width, int64_t lda) {
  static const bool off = [] { const char* e = getenv("HGT_BWD_SIMT"); return e && e[0] == '1'; }();
  if (off) return false;
  if (width % 8 || K % 16 || K < 64 || width < 16 || lda != K) return false;
  if (groups_overlap(h_groups, n_groups)) return false;
  int64_t rows = 0;
  for (int g = 0; g < n_groups; ++g) {
    rows += h_groups[g].m;
    for (int c = 0; c < h_groups[g].n_cblocks; ++c) {
      const hgt_lin_cblock& cb = h_cb[h_groups[g].cb_first + c];
      if (cb.out_off % 8 || cb.ld % 8) return false;
    }
  }
  return rows >= 512;                      // tiny problems (RTE tables, unit tests at c1 size) stay on the SIMT kernels
}

BwdLayout bwd_layout(const hgt_lin_group* h_groups, int n_groups, const hgt_lin_cblock* h_cb, int K, int width,
                     int64_t lda, int64_t dout_elems, bool have_dsplit, bool have_asplit, int impl, bool det) {
  BwdLayout L{};
  // impl 3 with a pre-split A (the forward kept only its bf16 hi half) needs the tensor cores, as impl 2 does
  L.tc = impl == 2 || (impl == 3 && have_asplit) ||
         ((impl == 0 || impl == 3) && bwd_tc_ok(h_groups, n_groups, h_cb, K, width, lda));
  L.one = L.tc && impl == 3;
  L.Kp = K;
  L.wpad = (width + BK - 1) / BK * BK;
  L.a_rows = 0;
  L.w_rows = 0;
  L.n_tasks = 0;
  for (int g = 0; g < n_groups; ++g) {
    L.a_rows = std::max<int64_t>(L.a_rows, h_groups[g].a_row0 + h_groups[g].m);
    L.w_rows = std::max<int64_t>(L.w_rows, (int64_t)h_groups[g].w_row0 + (int64_t)h_groups[g].n_cblocks * width);
    L.n_tasks += h_groups[g].n_cblocks;
  }
  L.wt_cols = (L.w_rows + width - 1) / width * L.wpad;
  size_t p = 0;
  auto take = [&](size_t bytes) { size_t o = p; p += hgt_align_up(bytes, 256); return o; };
  L.off_maps = take((size_t)(2 * L.n_tasks + 2 * n_groups + 2) * sizeof(CUtensorMap));
  L.off_tasks = take((size_t)std::max(L.n_tasks, 1) * sizeof(GcTask));
  L.off_gt0 = take((size_t)(n_groups + 1) * sizeof(int32_t));
  L.off_gfirst = take((size_t)(n_groups + 1) * sizeof(int64_t));
  if (L.tc) {
    L.off_dhi = take(have_dsplit ? 0 : (size_t)dout_elems * 2);
    L.off_dlo = take(have_dsplit || L.one ? 0 : (size_t)dout_elems * 2);
    L.off_ahi = take(have_asplit ? 0 : (size_t)L.a_rows * L.Kp * 2);
    L.off_alo = take(have_asplit || L.one ? 0 : (size_t)L.a_rows * L.Kp * 2);
    L.off_wthi = take((size_t)K * L.wt_cols * 2);
    L.off_wtlo = take(L.one ? 0 : (size_t)K * L.wt_cols * 2);
  }
  L.dw_chunk = 0;
  L.off_part = L.off_dbp = 0;
  if (det) {
    int64_t task_rows = 0;
    for (int g = 0; g < n_groups; ++g) task_rows += h_groups[g].m * h_groups[g].n_cblocks;
    L.dw_chunk = L.tc ? tc_dw_chunk(task_rows, width, K) : simt_det_chunk(task_rows);
    int64_t slots = 0, units = 0;
    for (int g = 0; g < n_groups; ++g) {
      slots += (h_groups[g].m + L.dw_chunk - 1) / L.dw_chunk * h_groups[g].n_cblocks;
      units += (h_groups[g].m + SPLIT_ROWS - 1) / SPLIT_ROWS * h_groups[g].n_cblocks;
    }
    L.off_part = take((size_t)slots * width * K * sizeof(float));
    L.off_dbp = take((size_t)std::max(slots, L.tc ? units : 0) * width * sizeof(float));
  }
  L.total = p + 256;
  return L;
}

// P: bf16 products per k-step (3: split, 1: hi only)
template <int BN, int P>
__global__ void __launch_bounds__(TILE_THREADS, 1) k_lin_dx_tc(const __grid_constant__ DxJob job, int n_tiles) {
  split3_tile<BN, false, BK, OUT_STAGE_BYTES, P>(job, n_tiles);
}
template <int BN, int P>
__global__ void __launch_bounds__(TILE_THREADS, 1) k_lin_dw_tc(const __grid_constant__ DwJob job, int n_tiles) {
  split3_tile<BN, true, BK, OUT_STAGE_BYTES, P>(job, n_tiles);
}

template <int BN, int P>
int launch_bwd(const DxJob& job, int tiles, cudaStream_t st) {
  const size_t smem = tile_smem_bytes<BN, BK, OUT_STAGE_BYTES, P>();
  HGT_CHECK_CUDA(cudaFuncSetAttribute(k_lin_dx_tc<BN, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_lin_dx_tc<BN, P><<<persistent_grid(tiles), TILE_THREADS, smem, st>>>(job, tiles);
  HGT_LAUNCH_CHECK();
  return 0;
}
template <int BN, int P>
int launch_bwd(const DwJob& job, int tiles, cudaStream_t st) {
  const size_t smem = tile_smem_bytes<BN, BK, OUT_STAGE_BYTES, P>();
  HGT_CHECK_CUDA(cudaFuncSetAttribute(k_lin_dw_tc<BN, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_lin_dw_tc<BN, P><<<persistent_grid(tiles), TILE_THREADS, smem, st>>>(job, tiles);
  HGT_LAUNCH_CHECK();
  return 0;
}

template <int BN, int P>
__global__ void __launch_bounds__(TILE_THREADS, 1) k_lin_dw_tc_det(const __grid_constant__ DwJobDet job, int n_tiles) {
  split3_tile<BN, true, BK, OUT_STAGE_BYTES, P>(job, n_tiles);
}
template <int BN, int P>
int launch_bwd(const DwJobDet& job, int tiles, cudaStream_t st) {
  const size_t smem = tile_smem_bytes<BN, BK, OUT_STAGE_BYTES, P>();
  HGT_CHECK_CUDA(cudaFuncSetAttribute(k_lin_dw_tc_det<BN, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_lin_dw_tc_det<BN, P><<<persistent_grid(tiles), TILE_THREADS, smem, st>>>(job, tiles);
  HGT_LAUNCH_CHECK();
  return 0;
}

// Tile width (64 / 128 / 256) x products (3 / 1) of one of the three tensor-core jobs; b_exact (dW jobs): P = 4.
template <class Job>
int launch_bwd_any(const Job& job, int tile_n, bool one, int tiles, cudaStream_t st, bool b_exact = false) {
  if constexpr (!std::is_same<Job, DxJob>::value) {
    if (b_exact && !one) {
      switch (tile_n) {
        case 64: return launch_bwd<64, 4>(job, tiles, st);
        case 128: return launch_bwd<128, 4>(job, tiles, st);
        default: return launch_bwd<256, 4>(job, tiles, st);
      }
    }
  }
  switch (tile_n) {
    case 64: return one ? launch_bwd<64, 1>(job, tiles, st) : launch_bwd<64, 3>(job, tiles, st);
    case 128: return one ? launch_bwd<128, 1>(job, tiles, st) : launch_bwd<128, 3>(job, tiles, st);
    default: return one ? launch_bwd<256, 1>(job, tiles, st) : launch_bwd<256, 3>(job, tiles, st);
  }
}

}  // namespace

extern "C" int hgt_act_split(const float* in, int64_t ld, int64_t rows, int32_t K, int32_t act, float* out_f32,
                             void* hi, void* lo, void* stream_) {
  HGT_REQUIRE(in && (out_f32 || hi) && (hi || !lo), "hgt_act_split: NULL argument");
  HGT_REQUIRE(act == 0 || act == 1, "hgt_act_split: act=%d (0 = identity, 1 = gelu)", act);
  HGT_REQUIRE(!hi || K % 8 == 0, "hgt_act_split: the bf16 split needs K %% 8 == 0 (K=%d)", K);
  if (rows == 0) return 0;
  const int Kp = (K + 3) / 4 * 4;
  const int64_t n = rows * (Kp / 4);
  k_act_split<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(
      in, ld, rows, K, Kp, act, out_f32, reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo));
  HGT_LAUNCH_CHECK();
  return 0;
}

namespace {

GcTask* d_tasks_ptr(char* base, const BwdLayout& L) { return reinterpret_cast<GcTask*>(base + L.off_tasks); }

int bwd_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks, int32_t K,
                        int32_t cb_width, int64_t lda, int64_t dout_elems, int32_t have_dout_split, int32_t have_a_split,
                        int32_t impl, size_t* out_bytes, bool det) {
  HGT_REQUIRE(out_bytes && (n_groups == 0 || (h_groups && h_cblocks)), "hgt_typed_linear_bwd_workspace_bytes: NULL argument");
  HGT_REQUIRE(n_groups >= 0, "hgt_typed_linear_bwd_workspace_bytes: n_groups=%d", n_groups);
  HGT_REQUIRE(impl >= 0 && impl <= 3, "hgt_typed_linear_bwd_workspace_bytes: unknown impl %d", impl);
  *out_bytes = bwd_layout(h_groups, n_groups, h_cblocks, K, cb_width, lda, dout_elems, have_dout_split != 0,
                          have_a_split != 0, impl, det).total;
  return 0;
}

// a16: A in bf16 (hgt_typed_linear_bwd_bf16a; A, a_hi_in and a_lo_in are then NULL, dA too).
int typed_linear_bwd(const float* dout, const void* dout_hi, const void* dout_lo, int64_t dout_elems,
                     const float* A, int64_t lda, const void* a_hi_in, const void* a_lo_in,
                     const float* W, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                     const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                     float* dA, int32_t accumulate_dA, const float* gelu_aux, float* dW, float* db,
                     int32_t impl, void* workspace, size_t workspace_bytes, void* stream_, bool det,
                     const __nv_bfloat16* a16 = nullptr) {
  cudaStream_t st = (cudaStream_t)stream_;
  HGT_REQUIRE(n_groups >= 0, "hgt_typed_linear_bwd: n_groups=%d", n_groups);
  HGT_REQUIRE(K > 0 && cb_width > 0 && (W || (a16 && !dA)), "hgt_typed_linear_bwd: K=%d cb_width=%d", K, cb_width);
  if (n_groups == 0) return 0;
  HGT_REQUIRE(groups && h_groups && h_cblocks, "hgt_typed_linear_bwd: NULL group tables");
  HGT_REQUIRE(impl >= 0 && impl <= 3, "hgt_typed_linear_bwd: unknown impl %d", impl);
  if (a16) a_hi_in = a16, a_lo_in = nullptr;
  // impl 3 reads only the hi halves, so a producer's split may come without its lo half; a bf16 A has no lo half
  const bool have_dsplit = dout_hi && (dout_lo || impl == 3),
             have_asplit = a_hi_in && (a_lo_in || impl == 3 || a16);
  HGT_REQUIRE(dout || have_dsplit, "hgt_typed_linear_bwd: neither dout nor its bf16 split given");
  const BwdLayout L = bwd_layout(h_groups, n_groups, h_cblocks, K, cb_width, lda, dout_elems, have_dsplit, have_asplit, impl,
                                 det);
  HGT_REQUIRE(workspace && workspace_bytes >= L.total, "hgt_typed_linear_bwd: workspace too small (%zu < %zu)",
              workspace_bytes, L.total);
  if (L.tc)
    HGT_REQUIRE(cb_width % 8 == 0 && K % 16 == 0 && K >= 64 && lda == K && !groups_overlap(h_groups, n_groups),
                "hgt_typed_linear_bwd: tensor-core path does not support K=%d cb_width=%d lda=%lld (or overlapping groups)",
                K, cb_width, (long long)lda);
  else
    HGT_REQUIRE(dout && (A || a16 || !dW), "hgt_typed_linear_bwd: the SIMT path needs fp32 dout and A");
  char* base = reinterpret_cast<char*>(hgt_align_up(reinterpret_cast<size_t>(workspace), 256));
  float* part = det ? reinterpret_cast<float*>(base + L.off_part) : nullptr;
  float* db_part = det ? reinterpret_cast<float*>(base + L.off_dbp) : nullptr;

  // ---- task table (one entry per group x column block) ----
  std::vector<GcTask> tasks(std::max(L.n_tasks, 1));
  std::vector<int32_t> gt0(n_groups + 1);
  std::vector<int64_t> gfirst(n_groups + 1);   // per group: first dA element (SIMT) or first dA tile (tensor cores)
  int nt = 0;
  int64_t elems = 0;
  for (int g = 0; g < n_groups; ++g) {
    gt0[g] = nt;
    gfirst[g] = elems;
    elems += h_groups[g].m * K;
    HGT_REQUIRE(h_groups[g].w_row0 % cb_width == 0, "hgt_typed_linear_bwd: w_row0=%d is not a multiple of cb_width=%d",
                h_groups[g].w_row0, cb_width);
    for (int c = 0; c < h_groups[g].n_cblocks; ++c, ++nt) {
      const hgt_lin_cblock& cb = h_cblocks[h_groups[g].cb_first + c];
      GcTask& t = tasks[nt];
      t.out_off = cb.out_off;
      t.ld = cb.ld;
      t.rows = h_groups[g].m;
      t.a_row0 = h_groups[g].a_row0;
      t.w_row = h_groups[g].w_row0 + c * cb_width;
      t.has_bias = h_groups[g].has_bias;
      t.first_unit = 0;
      t.n_chunks = 0;
      t.map_dout = 2 * nt;
      t.map_x = 2 * L.n_tasks + 2 * g;
      t.group = g;
      t.wt_col0 = (t.w_row / cb_width) * L.wpad;
      HGT_REQUIRE(dout_elems <= 0 || h_groups[g].m == 0 ||
                      cb.out_off + (h_groups[g].m - 1) * cb.ld + cb_width <= dout_elems,
                  "hgt_typed_linear_bwd: column block %d of group %d exceeds dout_elems", c, g);
    }
  }
  gt0[n_groups] = nt;
  gfirst[n_groups] = elems;
  // deterministic mode: sum of partial slots per W row (tasks in order, then slots in order); each row has one owner
  auto reduce_rows = [&](const float* src, int k_cols, int units_per_slot, int bias_only, float* out) -> int {
    const int64_t n = L.w_rows * k_cols;
    if (n == 0) return 0;
    k_reduce_rows<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, d_tasks_ptr(base, L), nt, cb_width, k_cols,
                                                                L.w_rows, units_per_slot, bias_only, out);
    HGT_LAUNCH_CHECK();
    return 0;
  };
  GcTask* d_tasks = reinterpret_cast<GcTask*>(base + L.off_tasks);
  int32_t* d_gt0 = reinterpret_cast<int32_t*>(base + L.off_gt0);
  int64_t* d_gfirst = reinterpret_cast<int64_t*>(base + L.off_gfirst);
  auto upload_tasks = [&]() -> int { return upload_bytes(d_tasks, tasks.data(), (size_t)nt * sizeof(GcTask), st); };
  // One upload of the contiguous workspace head [tensor maps (tensor cores only) | tasks | gt0 | gfirst]: the regions
  // are laid out in that order by bwd_layout; the alignment gaps between them are written as zeros.
  auto upload_head = [&](const std::vector<CUtensorMap>* maps) -> int {
    const size_t begin = maps ? L.off_maps : L.off_tasks;
    std::vector<unsigned char> img(L.off_gfirst + gfirst.size() * sizeof(int64_t) - begin, 0);
    if (maps) memcpy(img.data(), maps->data(), maps->size() * sizeof(CUtensorMap));
    memcpy(img.data() + (L.off_tasks - begin), tasks.data(), (size_t)nt * sizeof(GcTask));
    memcpy(img.data() + (L.off_gt0 - begin), gt0.data(), gt0.size() * sizeof(int32_t));
    memcpy(img.data() + (L.off_gfirst - begin), gfirst.data(), gfirst.size() * sizeof(int64_t));
    return upload_bytes(base + begin, img.data(), img.size(), st);
  };
  int rc;

  if (!L.tc) {
    // ---------------- SIMT fp32 path ----------------
    // the head carries the dX task table (first_unit unused there); dW uploads its own below
    if ((rc = upload_head(nullptr))) return rc;
    if (dA && det) {
      const int64_t n = L.a_rows * K;
      if (n > 0) {
        k_lin_dx_simt_det<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dout, W, d_tasks, d_gt0, groups, n_groups, L.a_rows,
                                                                       K, cb_width, gelu_aux, accumulate_dA, dA);
        HGT_LAUNCH_CHECK();
      }
    } else if (dA) {
      if (!accumulate_dA) HGT_CHECK_CUDA(cudaMemsetAsync(dA, 0, (size_t)L.a_rows * K * sizeof(float), st));
      if (elems > 0) {
        k_lin_dx_simt<<<(unsigned)((elems + 255) / 256), 256, 0, st>>>(dout, W, d_tasks, d_gt0, groups, n_groups, d_gfirst, K,
                                                                       cb_width, gelu_aux, dA);
        HGT_LAUNCH_CHECK();
      }
    }
    // db comes out of the dW kernel here, so it runs for db alone too
    if (dW || db) {
      const int n_tiles = (cb_width + 31) / 32, k_tiles = dW ? (K + 31) / 32 : 1;
      const int64_t chunk_rows = det ? L.dw_chunk : DW_SIMT_ROWS;
      int64_t units = 0;
      for (int t = 0; t < nt; ++t) {
        tasks[t].first_unit = (int32_t)units;
        tasks[t].n_chunks = (int32_t)((tasks[t].rows + chunk_rows - 1) / chunk_rows);
        units += (int64_t)tasks[t].n_chunks * n_tiles * k_tiles;
        HGT_REQUIRE(units < 2147483647ll, "hgt_typed_linear_bwd: too many units");
      }
      if ((rc = upload_tasks())) return rc;
      if (units > 0 && det) {
        if (a16)
          k_lin_dw_simt_det<<<(unsigned)units, 256, 0, st>>>(dout, a16, lda, d_tasks, nt, K, cb_width, n_tiles, k_tiles,
                                                             chunk_rows, dW ? part : nullptr, db ? db_part : nullptr);
        else
          k_lin_dw_simt_det<<<(unsigned)units, 256, 0, st>>>(dout, A, lda, d_tasks, nt, K, cb_width, n_tiles, k_tiles,
                                                             chunk_rows, dW ? part : nullptr, db ? db_part : nullptr);
        HGT_LAUNCH_CHECK();
        if (dW && (rc = reduce_rows(part, K, n_tiles * k_tiles, 0, dW))) return rc;
        if (db && (rc = reduce_rows(db_part, 1, n_tiles * k_tiles, 1, db))) return rc;
      } else if (units > 0) {
        if (a16)
          k_lin_dw_simt<<<(unsigned)units, 256, 0, st>>>(dout, a16, lda, d_tasks, nt, K, cb_width, n_tiles, k_tiles, dW, db);
        else
          k_lin_dw_simt<<<(unsigned)units, 256, 0, st>>>(dout, A, lda, d_tasks, nt, K, cb_width, n_tiles, k_tiles, dW, db);
        HGT_LAUNCH_CHECK();
      }
    }
    return 0;
  }

  // ---------------- tensor-core path ----------------
  __nv_bfloat16* d_hi = have_dsplit ? reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(dout_hi))
                                    : reinterpret_cast<__nv_bfloat16*>(base + L.off_dhi);
  __nv_bfloat16* d_lo = have_dsplit ? reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(dout_lo))
                                    : reinterpret_cast<__nv_bfloat16*>(base + L.off_dlo);
  __nv_bfloat16* a_hi = have_asplit ? reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a_hi_in))
                                    : reinterpret_cast<__nv_bfloat16*>(base + L.off_ahi);
  __nv_bfloat16* a_lo = have_asplit ? reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a_lo_in))
                                    : reinterpret_cast<__nv_bfloat16*>(base + L.off_alo);
  __nv_bfloat16* wt_hi = reinterpret_cast<__nv_bfloat16*>(base + L.off_wthi);
  __nv_bfloat16* wt_lo = reinterpret_cast<__nv_bfloat16*>(base + L.off_wtlo);
  // One product: the producers write no lo halves; the lo maps repeat the hi ones (never loaded, valid to prefetch).
  // The same for the lo half a bf16 A does not have.
  __nv_bfloat16* const d_lo_w = L.one ? nullptr : d_lo;
  __nv_bfloat16* const a_lo_w = L.one ? nullptr : a_lo;
  __nv_bfloat16* const wt_lo_w = L.one ? nullptr : wt_lo;
  if (L.one) d_lo = d_hi, a_lo = a_hi, wt_lo = wt_hi;
  if (a16) a_lo = a_hi;

  // 1. tensor maps: per task dOut hi/lo {cols = width, rows = m}; per group A hi/lo {cols = K, rows = m}; W^T hi/lo.
  //    They encode addresses only, so they go up with the task table before any kernel runs.
  std::vector<CUtensorMap> maps(2 * nt + 2 * n_groups + 2);
  for (int t = 0; t < nt; ++t) {
    if ((rc = make_map2(&maps[2 * t], d_hi + tasks[t].out_off, tasks[t].rows, cb_width, tasks[t].ld, 64))) return rc;
    if ((rc = make_map2(&maps[2 * t + 1], d_lo + tasks[t].out_off, tasks[t].rows, cb_width, tasks[t].ld, 64))) return rc;
  }
  for (int g = 0; g < n_groups; ++g) {
    if ((rc = make_map2(&maps[2 * nt + 2 * g], a_hi + h_groups[g].a_row0 * K, h_groups[g].m, K, K, 64))) return rc;
    if ((rc = make_map2(&maps[2 * nt + 2 * g + 1], a_lo + h_groups[g].a_row0 * K, h_groups[g].m, K, K, 64))) return rc;
  }
  const int map_wt = 2 * nt + 2 * n_groups;
  const int bn_box = pick_tile_n(K);                 // rows of the W^T box = dX tile width
  if ((rc = make_map2(&maps[map_wt], wt_hi, K, L.wt_cols, L.wt_cols, bn_box))) return rc;
  if ((rc = make_map2(&maps[map_wt + 1], wt_lo, K, L.wt_cols, L.wt_cols, bn_box))) return rc;
  CUtensorMap* d_maps = reinterpret_cast<CUtensorMap*>(base + L.off_maps);
  // the task table of the dOut split pass (the dX kernel reads only map indices / wt_col0 from it)
  int64_t split_units = 0;
  if (!have_dsplit) {
    for (int t = 0; t < nt; ++t) {
      tasks[t].first_unit = (int32_t)split_units;
      tasks[t].n_chunks = (int32_t)((tasks[t].rows + SPLIT_ROWS - 1) / SPLIT_ROWS);
      split_units += tasks[t].n_chunks;
      HGT_REQUIRE(split_units < 2147483647ll, "hgt_typed_linear_bwd: too many units");
    }
  }
  // the dX tiles of group g are [gfirst[g], gfirst[g + 1]); the prefix lives in the workspace, so a table may have any
  // number of groups
  const int dx_tile_n = pick_tile_n(K), dx_tiles_n = (K + dx_tile_n - 1) / dx_tile_n;
  for (int g = 0; g < n_groups; ++g) {
    gfirst[g + 1] = gfirst[g] + (h_groups[g].m + BM - 1) / BM * dx_tiles_n;
    HGT_REQUIRE(gfirst[g + 1] < 2147483647ll, "hgt_typed_linear_bwd: too many tiles");
  }
  if ((rc = upload_head(&maps))) return rc;

  // 2. dOut split (+ db) unless the producer already split it
  if (split_units > 0 && det) {
    k_split_colsum_det<<<(unsigned)split_units, 256, 0, st>>>(dout, d_tasks, nt, cb_width, d_hi, d_lo_w,
                                                              db ? db_part : nullptr);
    HGT_LAUNCH_CHECK();
    if (db && (rc = reduce_rows(db_part, 1, 1, 1, db))) return rc;
  } else if (split_units > 0) {
    k_split_colsum<<<(unsigned)split_units, 256, 0, st>>>(dout, d_tasks, nt, cb_width, d_hi, d_lo_w, db);
    HGT_LAUNCH_CHECK();
  }
  // 3. A split (dW needs it) unless saved by the forward
  if (dW && !have_asplit && L.a_rows > 0) {
    HGT_REQUIRE(A, "hgt_typed_linear_bwd: dW needs A or its bf16 split");
    const int64_t n = L.a_rows * (K / 4);
    k_act_split<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, lda, L.a_rows, K, K, 0, nullptr, a_hi, a_lo_w);
    HGT_LAUNCH_CHECK();
  }
  // 4. W^T split (dX)
  if (dA) {
    const int64_t n = (int64_t)K * L.wt_cols;
    k_wt_split<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, L.w_rows, K, cb_width, L.wpad, L.wt_cols, wt_hi, wt_lo_w);
    HGT_LAUNCH_CHECK();
  }

  // 5. dX
  if (dA) {
    // rows that no group covers keep a zero gradient
    if (!accumulate_dA) {
      std::vector<std::pair<int64_t, int64_t>> iv;
      for (int g = 0; g < n_groups; ++g)
        if (h_groups[g].m > 0) iv.emplace_back(h_groups[g].a_row0, h_groups[g].a_row0 + h_groups[g].m);
      std::sort(iv.begin(), iv.end());
      int64_t pos = 0;
      for (auto& p : iv) {
        if (p.first > pos) HGT_CHECK_CUDA(cudaMemsetAsync(dA + pos * K, 0, (size_t)(p.first - pos) * K * sizeof(float), st));
        pos = std::max(pos, p.second);
      }
    }
    const int64_t total = gfirst[n_groups];
    if (total > 0) {
      DxJob job;
      job.tile_n = dx_tile_n;
      job.n_tiles_n = dx_tiles_n;
      job.maps = d_maps;
      job.map_wt = map_wt;
      job.tasks = d_tasks;
      job.group_task0 = d_gt0;
      job.first_tile = d_gfirst;
      job.groups = groups;
      job.n_groups = n_groups;
      job.K_in = K;
      job.width = cb_width;
      job.dA = dA;
      job.accumulate = accumulate_dA;
      job.gelu_aux = gelu_aux;
      if ((rc = launch_bwd_any(job, job.tile_n, L.one, (int)total, st))) return rc;
    }
  }
  // 6. dW
  if (dW) {
    const int tile_n = pick_tile_n(K);
    const int m_tiles = (cb_width + BM - 1) / BM, n_tiles = (K + tile_n - 1) / tile_n;
    // chunk the reduction so that the grid has a few waves of CTAs
    int64_t task_rows = 0;
    for (int t = 0; t < nt; ++t) task_rows += tasks[t].rows;
    const int64_t chunk = tc_dw_chunk(task_rows, cb_width, K);
    int64_t units = 0;
    for (int t = 0; t < nt; ++t) {
      tasks[t].first_unit = (int32_t)units;
      tasks[t].n_chunks = (int32_t)((tasks[t].rows + chunk - 1) / chunk);
      units += (int64_t)tasks[t].n_chunks * m_tiles * n_tiles;
      HGT_REQUIRE(units < 2147483647ll, "hgt_typed_linear_bwd: too many units");
    }
    // the split / dX kernels enqueued above read the previous version of the table: stream order keeps them apart
    GcTask* d_tasks2 = d_tasks;
    if ((rc = upload_tasks())) return rc;
    if (units > 0) {
      DwJob job;
      job.maps = d_maps;
      job.tasks = d_tasks2;
      job.n_tasks = nt;
      job.K_in = K;
      job.width = cb_width;
      job.m_tiles = m_tiles;
      job.n_tiles = n_tiles;
      job.chunk_rows = (int)chunk;
      job.tile_n = tile_n;
      job.dW = dW;
      if (det) {
        DwJobDet dj;
        static_cast<DwJob&>(dj) = job;
        dj.part = part;
        if ((rc = launch_bwd_any(dj, tile_n, L.one, (int)units, st, a16 != nullptr))) return rc;
        if ((rc = reduce_rows(part, K, m_tiles * n_tiles, 0, dW))) return rc;
      } else {
        if ((rc = launch_bwd_any(job, tile_n, L.one, (int)units, st, a16 != nullptr))) return rc;
      }
    }
  }
  return 0;
}

}  // namespace

extern "C" int hgt_typed_linear_bwd_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups,
                                                    const hgt_lin_cblock* h_cblocks, int32_t K, int32_t cb_width,
                                                    int64_t lda, int64_t dout_elems, int32_t have_dout_split,
                                                    int32_t have_a_split, int32_t impl, size_t* out_bytes) {
  return bwd_workspace_bytes(h_groups, n_groups, h_cblocks, K, cb_width, lda, dout_elems, have_dout_split, have_a_split,
                             impl, out_bytes, false);
}

extern "C" int hgt_typed_linear_bwd(const float* dout, const void* dout_hi, const void* dout_lo, int64_t dout_elems,
                                    const float* A, int64_t lda, const void* a_hi_in, const void* a_lo_in,
                                    const float* W, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                    const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                                    float* dA, int32_t accumulate_dA, const float* gelu_aux, float* dW, float* db,
                                    int32_t impl, void* workspace, size_t workspace_bytes, void* stream_) {
  return typed_linear_bwd(dout, dout_hi, dout_lo, dout_elems, A, lda, a_hi_in, a_lo_in, W, K, cb_width, groups, h_groups,
                          n_groups, h_cblocks, dA, accumulate_dA, gelu_aux, dW, db, impl, workspace, workspace_bytes,
                          stream_, false);
}

extern "C" int hgt_typed_linear_bwd_det_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups,
                                                        const hgt_lin_cblock* h_cblocks, int32_t K, int32_t cb_width,
                                                        int64_t lda, int64_t dout_elems, int32_t have_dout_split,
                                                        int32_t have_a_split, int32_t impl, size_t* out_bytes) {
  return bwd_workspace_bytes(h_groups, n_groups, h_cblocks, K, cb_width, lda, dout_elems, have_dout_split, have_a_split,
                             impl, out_bytes, true);
}

extern "C" int hgt_typed_linear_bwd_det(const float* dout, const void* dout_hi, const void* dout_lo, int64_t dout_elems,
                                        const float* A, int64_t lda, const void* a_hi_in, const void* a_lo_in,
                                        const float* W, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                        const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                                        float* dA, int32_t accumulate_dA, const float* gelu_aux, float* dW, float* db,
                                        int32_t impl, void* workspace, size_t workspace_bytes, void* stream_) {
  return typed_linear_bwd(dout, dout_hi, dout_lo, dout_elems, A, lda, a_hi_in, a_lo_in, W, K, cb_width, groups, h_groups,
                          n_groups, h_cblocks, dA, accumulate_dA, gelu_aux, dW, db, impl, workspace, workspace_bytes,
                          stream_, true);
}

extern "C" int hgt_typed_linear_bwd_bf16a(const float* dout, int64_t dout_elems, const void* A, int64_t lda, int32_t K,
                                          int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                          int32_t n_groups, const hgt_lin_cblock* h_cblocks, float* dW, float* db,
                                          int32_t impl, void* workspace, size_t workspace_bytes, void* stream_) {
  HGT_REQUIRE(dout && (A || !dW), "hgt_typed_linear_bwd_bf16a: NULL argument");
  return typed_linear_bwd(dout, nullptr, nullptr, dout_elems, nullptr, lda, nullptr, nullptr, nullptr, K, cb_width, groups,
                          h_groups, n_groups, h_cblocks, nullptr, 0, nullptr, dW, db, impl, workspace, workspace_bytes,
                          stream_, false, static_cast<const __nv_bfloat16*>(A));
}

extern "C" int hgt_typed_linear_bwd_bf16a_det(const float* dout, int64_t dout_elems, const void* A, int64_t lda,
                                              int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                              const hgt_lin_group* h_groups, int32_t n_groups,
                                              const hgt_lin_cblock* h_cblocks, float* dW, float* db, int32_t impl,
                                              void* workspace, size_t workspace_bytes, void* stream_) {
  HGT_REQUIRE(dout && (A || !dW), "hgt_typed_linear_bwd_bf16a_det: NULL argument");
  return typed_linear_bwd(dout, nullptr, nullptr, dout_elems, nullptr, lda, nullptr, nullptr, nullptr, K, cb_width, groups,
                          h_groups, n_groups, h_cblocks, nullptr, 0, nullptr, dW, db, impl, workspace, workspace_bytes,
                          stream_, true, static_cast<const __nv_bfloat16*>(A));
}
