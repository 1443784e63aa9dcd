// Typed linear layers on the Hopper tensor cores (wgmma) with fp32-grade accuracy.
//
// fp32 operands are split into two bf16 terms, x = x_hi + x_lo (|x - x_hi - x_lo| <= 2^-17 |x|), and
//     A*W^T  ~=  A_hi*W_hi^T + A_hi*W_lo^T + A_lo*W_hi^T            (dropped term ~2^-18)
// is accumulated in ONE fp32 register accumulator by running three bf16 products per k-step inside the same
// tile: 3 tensor-core products at the bf16 rate instead of an fp32 FMA GEMM, error ~1e-5 relative —
// far inside the 1e-3 parity bar, where a single bf16 or tf32 product would not be.
//
// k_typed_linear_tc runs tcp::split3_tile (tc_ptx.cuh): a persistent grid of one CTA per SM walking the 128 x BN output tiles,
// a TMA producer warpgroup and two wgmma consumer warpgroups, both operands K-major.  At BN = 128 / 256 the k-blocks are 32
// wide (SWIZZLE_64B); their epilogue drains through asynchronous TMA tensor stores (tcp::store_tma), whose 64 KB of staging
// leaves a ring of 3 x 48 KB stages at BN = 256 and 5 x 32 KB at BN = 128.  BN = 64 keeps 64-wide k-blocks (SWIZZLE_128B,
// 4 stages) and the staged st.global epilogue: its k-blocks are short enough that halving them costs more in barrier
// waits than the deeper ring gains (measured on the d = 400 OAG shape).  Output tiles follow the same group / column-block tables
// as the SIMT kernel in linear.cu.  The output is fp32, bf16 (hgt_typed_linear[_presplit]_bf16), the planar 24-bit
// table format (hgt_typed_linear[_presplit]_t24) or the block-scaled bs16 format (hgt_typed_linear[_presplit]_bs16,
// include/hgt_b200.h): the same tile, rounded or encoded once as the epilogue stores it.
//
// One-product mode (P = 1: impl 3, or a presplit call with a_lo == NULL): the operands are rounded to bf16 (the hi half
// of the split, bitwise) and one bf16 product per k-step is accumulated, torch's "medium" float32 matmul precision.  Its
// stages hold {A_hi, W_hi} only; tiles, epilogues, barriers and tile order are those of P = 3.
//
// A operand: at BN = 128 / 256, hgt_typed_linear[_bf16] loads fp32 A with TMA (boxes of 32 floats x 128 rows,
// SWIZZLE_128B) and each consumer warpgroup splits its rows in shared memory, in place, into the bf16 halves its wgmma
// reads (tcp::split_a_slab): the same bits k_split_bf16 would write, so the result equals the presplit entry points' on
// hgt_act_split's halves, bitwise.  A k-block's fp32 A takes as many bytes as {A_hi, A_lo} did (twice A_hi's at P = 1),
// and there is no separate pass over A and no A halves in the workspace.  k_split_bf16 still splits A first for 64-column
// tiles (splits_a_first) and for an A that TMA cannot load as fp32 (base not 16-byte aligned, or lda % 4 != 0).  W is
// split once per call by k_split_bf16.
//
// bf16 A (hgt_typed_linear_bf16a): A is exactly its own hi half and its lo half is zero, so the x3 product loses its
// A_lo*W_hi term (tcp P = 2: A*W_hi + A*W_lo, two products per k-step) and P = 1 stays A*W_hi.  The products that remain
// run in P = 3's order and the dropped one adds exact zeros, so the output is bitwise that of the fp32 call on the
// widened A.  TMA loads A in place where its rows are 16-byte multiples (K % 8 == 0, lda % 8 == 0, base 16-byte aligned);
// otherwise (K = 129, 1169: the reference's input widths) k_pad_bf16 copies it first into zero-padded rows of Kp, the
// same place the fp32 path splits such an A into, in stream-ordered memory of its own.
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

using namespace tcp;

constexpr int kMaxGroups = 64;
template <int BN> constexpr int fwd_bk() { return BN == 64 ? 64 : 32; }    // k-block of the forward GEMM (P = 3)
template <int BN> constexpr bool fwd_tma_store() { return BN != 64; }      // tensor-store epilogue (FwdJob::store)
template <int BN> constexpr uint32_t fwd_out_stage() { return fwd_tma_store<BN>() ? TMA_STAGE_BYTES : OUT_STAGE_BYTES; }

// ---- fp32 -> (bf16 hi, bf16 lo) split; lo == NULL: hi only -------------------------------------------
__global__ void k_split_bf16(const float* __restrict__ in, int64_t ld_in, int64_t rows, int K, int Kp,
                             __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const int vec_per_row = Kp / 4;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= rows * vec_per_row) return;
  int64_t r = i / vec_per_row;
  int c = (int)(i - r * vec_per_row) * 4;
  float v[4];
  const float* src = in + r * ld_in + c;
  if (c + 3 < K && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
    float4 t = *reinterpret_cast<const float4*>(src);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = (c + j < K) ? src[j] : 0.f;
  }
  __nv_bfloat16 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = __float2bfloat16_rn(v[j]);
    l[j] = __float2bfloat16_rn(v[j] - __bfloat162float(h[j]));
  }
  *reinterpret_cast<uint2*>(hi + r * Kp + c) = *reinterpret_cast<uint2*>(h);
  if (lo) *reinterpret_cast<uint2*>(lo + r * Kp + c) = *reinterpret_cast<uint2*>(l);
}

// ---- bf16 [rows, K] (row stride ld_in) -> [rows, Kp], columns K .. Kp - 1 zero --------------------------------------
__global__ void k_pad_bf16(const __nv_bfloat16* __restrict__ in, int64_t ld_in, int64_t rows, int K, int Kp,
                           __nv_bfloat16* __restrict__ out) {
  const int vec_per_row = Kp / 4;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= rows * vec_per_row) return;
  int64_t r = i / vec_per_row;
  int c = (int)(i - r * vec_per_row) * 4;
  const __nv_bfloat16* src = in + r * ld_in + c;
  __nv_bfloat16 v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = (c + j < K) ? src[j] : __float2bfloat16_rn(0.f);
  *reinterpret_cast<uint2*>(out + r * Kp + c) = *reinterpret_cast<uint2*>(v);
}

// Columns col .. col + 3 of an output row: fp32, or bf16 rounded to nearest-even.  aligned: p is 4-element aligned.
__device__ __forceinline__ void store4(float* p, float4 v, bool aligned) {
  if (aligned) {
    *reinterpret_cast<float4*>(p) = v;
  } else if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) {
    *reinterpret_cast<float2*>(p) = make_float2(v.x, v.y);
    *reinterpret_cast<float2*>(p + 2) = make_float2(v.z, v.w);
  } else {
    p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w;
  }
}
__device__ __forceinline__ void store4(__nv_bfloat16* p, float4 v, bool aligned) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  if (aligned) {
    *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  } else {
    p[0] = a.x; p[1] = a.y; p[2] = b.x; p[3] = b.y;
  }
}
// 24-bit tables: hi halves at `hi`, lo bytes at `lo`.  aligned: hi 8-byte and lo 4-byte aligned.
__device__ __forceinline__ void store4_t24(unsigned char* hi, unsigned char* lo, float4 v, bool aligned) {
  uint32_t h01, l01, h23, l23;
  t24_pair(make_float2(v.x, v.y), h01, l01);
  t24_pair(make_float2(v.z, v.w), h23, l23);
  if (aligned) {
    *reinterpret_cast<uint2*>(hi) = make_uint2(h01, h23);
    *reinterpret_cast<uint32_t*>(lo) = __byte_perm(l01, l23, 0x5410);
  } else {
    const uint32_t h[4] = {h01 & 0xffffu, h01 >> 16, h23 & 0xffffu, h23 >> 16}, l[4] = {l01 & 0xffu, l01 >> 8, l23 & 0xffu, l23 >> 8};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      hi[2 * i] = (unsigned char)h[i];
      hi[2 * i + 1] = (unsigned char)(h[i] >> 8);
      lo[i] = (unsigned char)l[i];
    }
  }
}

// bs16 tables: columns col .. col + 3 of a row (a quarter of a 16-column block, whose other quarters the neighbouring
// lanes of an aligned quad hold; every lane of the warp calls this) as mantissas at `m` and, from the quad's first lane,
// the block's scale at `s`.  store: the row and the columns lie inside the output.
__device__ __forceinline__ void store4_bs16(unsigned char* m, unsigned char* s, float4 v, bool store, int lane) {
  const uint32_t a = hgt_bs16_quad_amax(max(max(hgt_abs_bits(v.x), hgt_abs_bits(v.y)),
                                            max(hgt_abs_bits(v.z), hgt_abs_bits(v.w))));
  float r;
  const uint32_t sb = hgt_bs16_scale(a, r);
  if (!store) return;
  *reinterpret_cast<uint2*>(m) = make_uint2(hgt_bs16_pack(v.x, v.y, r, sb), hgt_bs16_pack(v.z, v.w, r, sb));
  if ((lane & 3) == 0) *reinterpret_cast<uint16_t*>(s) = (uint16_t)sb;
}

// ---- the GEMM: out_cb[m, n] = A[a_row0 + m, :] . W[w_row0 + cb * cb_width + n, :] (+ bias) ------------------------------
// Rows of a tile past the group and columns past the column block are computed on neighbouring (or zero-filled) operand
// rows and not stored.
// AF: a_hi is the fp32 A map (box {32, 128 rows}, one or two per k-block) and a_lo repeats it.
template <class OutT, bool AF = false>
struct FwdJob {
  CUtensorMap a_hi, a_lo, w_hi, w_lo;      // A box {fwd_bk, 128 rows}, W box {fwd_bk, tile_n rows}
  const float* bias;
  const hgt_lin_group* groups;
  const hgt_lin_cblock* cblocks;
  OutT* out;
  float* out32;                            // table jobs (24-bit, bs16): column blocks with out_off < t24_off are fp32 at
  int64_t t24_off;                         // out32 + out_off, the others in the table at `out`, logical offset out_off - t24_off
  const CUtensorMap* out_maps;             // BN = 128 / 256: output map(s) of (group g, column block cb) at map_first[g] + cb
  int n_groups, cb_width, k_blocks, tile_n, n_tiles_n;
  int32_t first_tile[kMaxGroups + 1];
  int32_t map_first[kMaxGroups];

  struct Tile {
    int a_row, w_row, cols, m0, n0;
    int64_t rows, ld;
    OutT* out;
    float* out32;                          // table jobs: the tile's fp32 output, or NULL
    unsigned char *hi, *lo;                // 24-bit tables: the planes' bytes of the tile's element (0, 0); bs16: its
                                           // mantissa and its block's scale
    const float* bias;
    const CUtensorMap* map;
  };

  __device__ int decode(int tile, Tile& t) const {
    int g = 0;
    while (g + 1 < n_groups && tile >= first_tile[g + 1]) ++g;
    const hgt_lin_group grp = groups[g];
    int local = tile - first_tile[g];
    const int per_m = grp.n_cblocks * n_tiles_n;
    const int mt = local / per_m;
    local -= mt * per_m;
    const int cb = local / n_tiles_n;
    const int n0 = (local - cb * n_tiles_n) * tile_n;
    const hgt_lin_cblock cblk = cblocks[grp.cb_first + cb];
    const int64_t m0 = (int64_t)mt * BM;
    t.a_row = (int)(grp.a_row0 + m0);
    t.w_row = grp.w_row0 + cb * cb_width + n0;
    t.cols = cb_width - n0;
    t.rows = grp.m - m0;
    t.ld = cblk.ld;
    if constexpr (is_t24<OutT>()) {
      const int64_t off = cblk.out_off + m0 * cblk.ld + n0;
      t.out32 = cblk.out_off < t24_off ? out32 + off : nullptr;
      const hgt_t24_at e(out, off - t24_off, cblk.ld);
      t.hi = e.hi;
      t.lo = e.lo;
    } else if constexpr (is_bs16<OutT>()) {
      const int64_t off = cblk.out_off + m0 * cblk.ld + n0;
      t.out32 = cblk.out_off < t24_off ? out32 + off : nullptr;
      const hgt_bs16_at e(out, off - t24_off, cblk.ld);
      t.hi = e.m;
      t.lo = e.s;
    } else {
      t.out = out + cblk.out_off + m0 * cblk.ld + n0;
    }
    t.bias = (grp.has_bias && bias) ? bias + t.w_row : nullptr;
    t.m0 = (int)m0;
    t.n0 = n0;
    t.map = out_maps + out_maps_per_block<OutT>() * (map_first[g] + cb);
    return k_blocks;
  }
  __device__ void prefetch(const Tile&) const {
    prefetch_map(&a_hi); prefetch_map(&a_lo); prefetch_map(&w_hi); prefetch_map(&w_lo);
  }
  template <int BN, int KB, int P>
  __device__ void load(const Tile& t, int kb, uint32_t sa, uint32_t bar) const {
    constexpr uint32_t A = a_bytes<KB>(), B = b_offset<KB, P, AF>();
    const int k = kb * KB;
    if constexpr (AF) {
#pragma unroll
      for (int j = 0; j < KB / 32; ++j) tma_load_2d(sa + j * A32_BOX, &a_hi, k + 32 * j, t.a_row, bar);
    } else {
      tma_load_2d(sa, &a_hi, k, t.a_row, bar);
      if constexpr (has_a_lo<P>()) tma_load_2d(sa + A, &a_lo, k, t.a_row, bar);
    }
    tma_load_2d(sa + B, &w_hi, k, t.w_row, bar);
    if constexpr (has_b_lo<P>()) tma_load_2d(sa + B + BN * KB * 2, &w_lo, k, t.w_row, bar);
  }
  // OutT (or fp32 T, the fp32 blocks of a 24-bit job) at o, the tile's element (0, 0)
  template <int BN, class T, class Pair>
  __device__ void store_plain(const Tile& t, T* o, const float* acc, float* stage, int c, int wq, int lane,
                              Pair pair) const {
    o += (int64_t)(64 * c) * t.ld;
    const int64_t rows = t.rows - 64 * c, ld = t.ld;
    const int cols = t.cols;
    const uintptr_t align = reinterpret_cast<uintptr_t>(o) | (uintptr_t)(ld * sizeof(T));
    if constexpr (fwd_tma_store<BN>()) {
      if ((align & 15) == 0) {
        store_tma<BN, T>(acc, reinterpret_cast<unsigned char*>(stage), c, wq, lane, pair, t.map, t.n0, t.m0 + 64 * c,
                         cols);
        return;
      }
      if (wq == 0 && lane == 0) bulk_wait_read<0>();          // store_staged reuses the tensor stores' buffers
    }
    const bool vec4 = (align & (4 * sizeof(T) - 1)) == 0;
    store_staged<BN>(acc, stage, c, wq, lane, pair, [&](int r, int col, float4 v) {
      if (r < rows && col < cols) store4(o + r * ld + col, v, vec4);
    });
  }
  // BN = 128 / 256: asynchronous TMA tensor stores (tcp::store_tma) where the destination rows are 16-byte aligned, so
  // the stores overlap the next tile's products.  Otherwise, and at BN = 64, through shared memory with whole row segments
  // per warp (tcp::store_staged).  cols is a multiple of 16, so a 4-column group is either inside the column block or
  // past it.  Both paths add the bias in fp32 and round once, so they write the same bits.
  template <int BN>
  __device__ void store(const Tile& t, const float* acc, float* stage, int c, int wq, int lane) const {
    const float* b = t.bias;
    const int cols = t.cols;
    auto pair = [&](int, int col, float v0, float v1) {
      if (b && col < cols) v0 += __ldg(b + col), v1 += __ldg(b + col + 1);
      return make_float2(v0, v1);
    };
    if constexpr (is_t24<OutT>()) {
      if (t.out32) {
        store_plain<BN>(t, t.out32, acc, stage, c, wq, lane, pair);
        return;
      }
      const int64_t rows = t.rows - 64 * c;
      const int64_t rb = 3 * t.ld;                            // row stride in bytes
      unsigned char* hi = t.hi + 64 * c * rb;
      unsigned char* lo = t.lo + 64 * c * rb;
      if constexpr (fwd_tma_store<BN>()) {
        if (((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo) | (uintptr_t)rb) & 15) == 0) {
          store_tma<BN, OutT>(acc, reinterpret_cast<unsigned char*>(stage), c, wq, lane, pair, t.map, t.n0,
                              t.m0 + 64 * c, cols);
          return;
        }
        if (wq == 0 && lane == 0) bulk_wait_read<0>();
      }
      const bool vec4 = ((reinterpret_cast<uintptr_t>(hi) | (uintptr_t)rb) & 7) == 0 &&
                        ((reinterpret_cast<uintptr_t>(lo) | (uintptr_t)rb) & 3) == 0;
      store_staged<BN>(acc, stage, c, wq, lane, pair, [&](int r, int col, float4 v) {
        if (r < rows && col < cols) store4_t24(hi + r * rb + 2 * col, lo + r * rb + col, v, vec4);
      });
    } else if constexpr (is_bs16<OutT>()) {
      if (t.out32) {
        // the fp32 boxes fill whole buffers: the scale box of a previous bs16 tile must have been read out
        if (fwd_tma_store<BN>() && wq == 0 && lane == 0) bulk_wait_read<0>();
        store_plain<BN>(t, t.out32, acc, stage, c, wq, lane, pair);
        return;
      }
      const int64_t rows = t.rows - 64 * c;
      const int64_t rb = hgt_bs16_row_bytes(t.ld);             // row stride in bytes, a multiple of 16
      unsigned char* m = t.hi + 64 * c * rb;
      unsigned char* sc = t.lo + 64 * c * rb;
      if constexpr (fwd_tma_store<BN>()) {
        // k_out_maps' alignment rule, and a tile whose scale box lies inside the column block (a box that TMA clips at
        // a column that is not a 16-byte multiple wrote wrong scales)
        if (((reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(sc)) & 15) == 0 && cols >= BN) {
          store_tma<BN, OutT>(acc, reinterpret_cast<unsigned char*>(stage), c, wq, lane, pair, t.map, t.n0,
                              t.m0 + 64 * c, cols);
          return;
        }
        if (wq == 0 && lane == 0) bulk_wait_read<0>();
      }
      store_staged<BN>(acc, stage, c, wq, lane, pair, [&](int r, int col, float4 v) {
        store4_bs16(m + r * rb + 2 * col, sc + r * rb + 2 * (col / 16), v, r < rows && col < cols, lane);
      });
    } else {
      store_plain<BN>(t, t.out, acc, stage, c, wq, lane, pair);
    }
  }
};

template <int BN, class OutT, int P = 3, int KB = fwd_bk<BN>(), bool AF = false>
__global__ void __launch_bounds__(TILE_THREADS, 1)
    k_typed_linear_tc(const __grid_constant__ FwdJob<OutT, AF> job, int n_tiles) {
  split3_tile<BN, false, KB, fwd_out_stage<BN>(), P, AF>(job, n_tiles);
}

// ---- output tensor maps of the tensor-store epilogue ----------------------------------------------------------------
// One map per (group, column block) of a launch: base out + out_off, rows = the group's m, columns = cb_width, row stride
// ld.  The column-block table lives on the device, so the maps are built there: a copy of a host-encoded template (element
// type, box, swizzle, columns) with the address, the row count and the row stride replaced.  Maps of blocks whose rows
// are not 16-byte aligned are left unwritten; their tiles take the staged epilogue.  24-bit tables have two maps per block,
// the hi plane's (from `tmpl`) and the lo plane's (from `tmpl_lo`), at the planes' bytes with row stride 3 ld bytes; the
// fp32 blocks of a 24-bit job one (from `tmpl_f32`).
struct MapFirst {
  int32_t v[kMaxGroups];
};

__device__ __forceinline__ void put_map(CUtensorMap* m, const CUtensorMap& tmpl, const void* base, int64_t rows,
                                        uint64_t stride) {
#pragma unroll
  for (int i = 0; i < 8; ++i) reinterpret_cast<uint4*>(m)[i] = reinterpret_cast<const uint4*>(&tmpl)[i];
  const uint64_t gm = (uint64_t)__cvta_generic_to_global(m);
  asm volatile("tensormap.replace.tile.global_address.global.b1024.b64 [%0], %1;" ::"l"(gm), "l"(base) : "memory");
  asm volatile("tensormap.replace.tile.global_dim.global.b1024.b32 [%0], 1, %1;" ::"l"(gm), "r"((uint32_t)rows)
               : "memory");
  asm volatile("tensormap.replace.tile.global_stride.global.b1024.b64 [%0], 0, %1;" ::"l"(gm), "l"(stride) : "memory");
}

template <class OutT>
__global__ void k_out_maps(const __grid_constant__ CUtensorMap tmpl, const __grid_constant__ CUtensorMap tmpl_lo,
                           const __grid_constant__ CUtensorMap tmpl_f32, const hgt_lin_group* __restrict__ groups,
                           const hgt_lin_cblock* __restrict__ cblocks, OutT* out, float* out32, int64_t t24_off,
                           const MapFirst first, CUtensorMap* maps) {
  const hgt_lin_group grp = groups[blockIdx.x];
  for (int cb = threadIdx.x; cb < grp.n_cblocks; cb += blockDim.x) {
    const hgt_lin_cblock cblk = cblocks[grp.cb_first + cb];
    CUtensorMap* m = maps + out_maps_per_block<OutT>() * (first.v[blockIdx.x] + cb);
    if (grp.m <= 0) continue;
    if (is_table<OutT>() && cblk.out_off < t24_off) {
      const float* base = out32 + cblk.out_off;
      const uint64_t stride = (uint64_t)cblk.ld * 4;
      if (((reinterpret_cast<uintptr_t>(base) | stride) & 15) != 0) continue;
      put_map(m, tmpl_f32, base, grp.m, stride);
    } else if constexpr (is_t24<OutT>()) {
      const hgt_t24_at e(out, cblk.out_off - t24_off, cblk.ld);
      const uint64_t stride = 3 * (uint64_t)cblk.ld;
      if (((reinterpret_cast<uintptr_t>(e.hi) | reinterpret_cast<uintptr_t>(e.lo) | stride) & 15) != 0) continue;
      put_map(m, tmpl, e.hi, grp.m, stride);
      put_map(m + 1, tmpl_lo, e.lo, grp.m, stride);
    } else if constexpr (is_bs16<OutT>()) {
      const hgt_bs16_at e(out, cblk.out_off - t24_off, cblk.ld);
      const uint64_t stride = (uint64_t)hgt_bs16_row_bytes(cblk.ld);
      if (((reinterpret_cast<uintptr_t>(e.m) | reinterpret_cast<uintptr_t>(e.s)) & 15) != 0) continue;
      put_map(m, tmpl, e.m, grp.m, stride);
      put_map(m + 1, tmpl_lo, e.s, grp.m, stride);
    } else {
      OutT* base = out + cblk.out_off;
      const uint64_t stride = (uint64_t)cblk.ld * sizeof(OutT);
      if (((reinterpret_cast<uintptr_t>(base) | stride) & 15) != 0) continue;
      put_map(m, tmpl, base, grp.m, stride);
    }
  }
  asm volatile("fence.proxy.tensormap::generic.release.gpu;" ::: "memory");
}

// ---- host side ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
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

// bf16 [rows, Kp] at row stride ld elements (default Kp), boxes of kb columns x box_rows rows.
int make_map(CUtensorMap* m, const void* base, int64_t rows, int Kp, int box_rows, int kb, int64_t ld = 0) {
  EncodeTiledFn fn = get_encode_fn();
  HGT_REQUIRE(fn != nullptr, "hgt_typed_linear: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(ld ? ld : Kp) * 2};
  cuuint32_t box[2] = {(cuuint32_t)kb, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, kb == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HGT_REQUIRE(r == CUDA_SUCCESS, "hgt_typed_linear: cuTensorMapEncodeTiled failed (%d) rows=%lld Kp=%d box=%d",
              (int)r, (long long)rows, Kp, box_rows);
  return 0;
}

// fp32 A as the GEMM loads it (AF): K columns at row stride lda, boxes of 32 floats (128 bytes, SWIZZLE_128B) x 128 rows.
// TMA zero-fills columns k >= K and rows past `rows`, as the split's padding to Kp did.  Needs A 16-byte aligned and
// lda % 4 == 0 (a_fp32_loadable).
int make_map_f32(CUtensorMap* m, const float* base, int64_t rows, int K, int64_t lda) {
  EncodeTiledFn fn = get_encode_fn();
  HGT_REQUIRE(fn != nullptr, "hgt_typed_linear: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)lda * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)BM};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HGT_REQUIRE(r == CUDA_SUCCESS, "hgt_typed_linear: cuTensorMapEncodeTiled (fp32 A) failed (%d) rows=%lld K=%d lda=%lld",
              (int)r, (long long)rows, K, (long long)lda);
  return 0;
}

bool a_fp32_loadable(const float* A, int64_t lda) {
  return A && (reinterpret_cast<uintptr_t>(A) & 15) == 0 && lda % 4 == 0;
}

// Template of the output maps: `cb_width` columns of `elem`-byte elements, boxes of 128 bytes x 64 rows with SWIZZLE_128B
// (the layout tcp::store_tma stages), or of 64 bytes with SWIZZLE_64B (elem = 1: the lo plane of a 24-bit table).
// scale_box > 0: the scale plane of a bs16 table, cb_width / 16 bf16 per row, unswizzled boxes of scale_box x 64.
// `dummy` (16-byte aligned) and the row count / stride are placeholders that k_out_maps replaces.
int make_out_template(CUtensorMap* m, void* dummy, int cb_width, int elem, int scale_box = 0) {
  EncodeTiledFn fn = get_encode_fn();
  HGT_REQUIRE(fn != nullptr, "hgt_typed_linear: cuTensorMapEncodeTiled not available from the driver");
  const int cols = scale_box ? cb_width / 16 : cb_width;
  cuuint64_t dims[2] = {(cuuint64_t)cols, 64};
  cuuint64_t strides[1] = {(cuuint64_t)hgt_align_up((size_t)cols * elem, 16)};
  cuuint32_t box[2] = {scale_box ? (cuuint32_t)scale_box : elem == 1 ? 64u : 128 / (cuuint32_t)elem, 64};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType type = elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : elem == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = fn(m, type, 2, dummy, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  scale_box ? CU_TENSOR_MAP_SWIZZLE_NONE
                            : elem == 1 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HGT_REQUIRE(r == CUDA_SUCCESS, "hgt_typed_linear: cuTensorMapEncodeTiled (output) failed (%d) cb_width=%d", (int)r,
              cb_width);
  return 0;
}

int64_t n_out_maps(const hgt_lin_group* h_groups, int n_groups) {
  int64_t n = 0;
  for (int g = 0; g < n_groups; ++g) n += h_groups[g].n_cblocks;
  return n;
}

void extents(const hgt_lin_group* h_groups, int n_groups, int cb_width, int64_t* a_rows, int64_t* w_rows) {
  *a_rows = 0;
  *w_rows = 0;
  for (int g = 0; g < n_groups; ++g) {
    int64_t a = h_groups[g].a_row0 + h_groups[g].m;
    int64_t w = (int64_t)h_groups[g].w_row0 + (int64_t)h_groups[g].n_cblocks * cb_width;
    if (a > *a_rows) *a_rows = a;
    if (w > *w_rows) *w_rows = w;
  }
}

// Operands of one launch: A as fp32 (a32, lda; AF) or as bf16 halves (a_hi, a_lo), W as bf16 halves.  Halves are K-major
// at row stride Kp (A's at a_ld where that is set: a bf16 A read in place); a lo pointer is NULL where P has no lo half.
struct FwdOps {
  const float* a32;
  int64_t lda, a_ld = 0;
  const __nv_bfloat16 *a_hi, *a_lo, *w_hi, *w_lo;
  int64_t a_rows, w_rows;
  int K, Kp;
  float* out32;                           // 24-bit jobs: see FwdJob
  int64_t t24_off;
};

// The tensor maps and the k-block count follow the kernel's k-block KB.  At P = 1 (and for A under AF) the lo maps repeat
// the hi ones (the kernel does not load them; they stay valid for its prefetches).
template <int BN, class OutT, int P = 3, int KB = fwd_bk<BN>(), bool AF = false>
int launch_fwd(FwdJob<OutT, AF>& job, const FwdOps& ops, int tiles, cudaStream_t st) {
  int rc;
  if constexpr (AF) {
    if ((rc = make_map_f32(&job.a_hi, ops.a32, ops.a_rows, ops.K, ops.lda))) return rc;
    job.a_lo = job.a_hi;
  } else {
    if ((rc = make_map(&job.a_hi, ops.a_hi, ops.a_rows, ops.Kp, BM, KB, ops.a_ld))) return rc;
    if ((rc = make_map(&job.a_lo, has_a_lo<P>() ? ops.a_lo : ops.a_hi, ops.a_rows, ops.Kp, BM, KB, ops.a_ld))) return rc;
  }
  if ((rc = make_map(&job.w_hi, ops.w_hi, ops.w_rows, ops.Kp, BN, KB))) return rc;
  if ((rc = make_map(&job.w_lo, has_b_lo<P>() ? ops.w_lo : ops.w_hi, ops.w_rows, ops.Kp, BN, KB))) return rc;
  job.k_blocks = (ops.Kp + KB - 1) / KB;
  if constexpr (fwd_tma_store<BN>()) {
    CUtensorMap tmpl, tmpl_lo, tmpl_f32;
    MapFirst first;
    void* dummy = const_cast<CUtensorMap*>(job.out_maps);
    // 24-bit tables: the hi plane's u16 elements as bf16 (the maps only move bytes), the lo plane's u8, fp32 blocks;
    // bs16 tables: the int16 mantissas as bf16, fp32 blocks
    if ((rc = make_out_template(&tmpl, dummy, job.cb_width, is_table<OutT>() ? 2 : (int)sizeof(OutT)))) return rc;
    tmpl_lo = tmpl_f32 = tmpl;
    if (is_t24<OutT>() && (rc = make_out_template(&tmpl_lo, dummy, job.cb_width, 1))) return rc;
    if (is_bs16<OutT>() && (rc = make_out_template(&tmpl_lo, dummy, job.cb_width, 2, BN / 16))) return rc;
    if (is_table<OutT>() && (rc = make_out_template(&tmpl_f32, dummy, job.cb_width, 4))) return rc;
    for (int g = 0; g < job.n_groups; ++g) first.v[g] = job.map_first[g];
    k_out_maps<OutT><<<job.n_groups, 64, 0, st>>>(tmpl, tmpl_lo, tmpl_f32, job.groups, job.cblocks, job.out, job.out32,
                                                  job.t24_off, first, const_cast<CUtensorMap*>(job.out_maps));
    HGT_LAUNCH_CHECK();
  }
  const size_t smem = tile_smem_bytes<BN, KB, fwd_out_stage<BN>(), P, AF>();
  HGT_CHECK_CUDA(cudaFuncSetAttribute(k_typed_linear_tc<BN, OutT, P, KB, AF>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_typed_linear_tc<BN, OutT, P, KB, AF><<<persistent_grid(tiles), TILE_THREADS, smem, st>>>(job, tiles);
  HGT_LAUNCH_CHECK();
  return 0;
}

// Fills the job's tile tables and launches the instance for its tile width, product count and A operand.  a_exact: A is
// bf16 (no lo half), and one == false runs P = 2.
template <class OutT, bool AF>
int run_fwd(const FwdOps& ops, const float* bias, int32_t cb_width, const hgt_lin_group* groups,
            const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* cblocks, OutT* out,
            CUtensorMap* out_maps, bool one, cudaStream_t st, bool a_exact = false) {
  FwdJob<OutT, AF> job;
  job.tile_n = pick_tile_n(cb_width);
  job.n_tiles_n = (cb_width + job.tile_n - 1) / job.tile_n;
  int64_t total = 0, maps = 0;
  for (int g = 0; g < n_groups; ++g) {
    job.map_first[g] = (int32_t)maps;
    maps += h_groups[g].n_cblocks;
    job.first_tile[g] = (int32_t)total;
    total += (h_groups[g].m + BM - 1) / BM * h_groups[g].n_cblocks * job.n_tiles_n;
    HGT_REQUIRE(total < 2147483647ll, "hgt_typed_linear(tc): too many tiles");
  }
  job.first_tile[n_groups] = (int32_t)total;
  if (total == 0) return 0;
  job.bias = bias;
  job.groups = groups;
  job.cblocks = cblocks;
  job.out = out;
  job.out32 = ops.out32;
  job.t24_off = ops.t24_off;
  job.out_maps = out_maps;
  job.n_groups = n_groups;
  job.cb_width = cb_width;
  const int tiles = (int)total;
  // 64-column tiles read A split by k_split_bf16 (tc_run): only the presplit instances exist for them
  if constexpr (AF) HGT_REQUIRE(job.tile_n != 64, "hgt_typed_linear(tc): no fp32-A kernel for 64-column tiles");
  if constexpr (!AF && std::is_same<OutT, float>::value) {
    if (a_exact && !one) {
      switch (job.tile_n) {
        case 64: return launch_fwd<64, OutT, 2, fwd_bk<64>()>(job, ops, tiles, st);
        case 128: return launch_fwd<128, OutT, 2, fwd_bk<128>()>(job, ops, tiles, st);
        default: return launch_fwd<256, OutT, 2, fwd_bk<256>()>(job, ops, tiles, st);
      }
    }
  }
  HGT_REQUIRE(!a_exact || one, "hgt_typed_linear_bf16a(tc): fp32 output only");
  if (one) {
    // k-block of the one-product kernel at BN = 128 / 256 (DESIGN.md §5.2): 32 (SWIZZLE_64B, as at P = 3) for fp32 A,
    // whose 64-wide stages would leave a ring of two at BN = 256; 64 (SWIZZLE_128B) for presplit A.  HGT_TC_P1_KB=32 or
    // 64 selects one for both, for A/B measurements.
    static const int kb_env = [] {
      const char* e = getenv("HGT_TC_P1_KB");
      return !e ? 0 : (e[0] == '3' && e[1] == '2') ? 32 : (e[0] == '6' && e[1] == '4') ? 64 : 0;
    }();
    const bool kb32 = kb_env ? kb_env == 32 : AF;
    switch (job.tile_n) {
      case 64:
        if constexpr (!AF) return launch_fwd<64, OutT, 1, 64>(job, ops, tiles, st);
        return 1;
      case 128:
        return kb32 ? launch_fwd<128, OutT, 1, 32, AF>(job, ops, tiles, st)
                    : launch_fwd<128, OutT, 1, 64, AF>(job, ops, tiles, st);
      default:
        return kb32 ? launch_fwd<256, OutT, 1, 32, AF>(job, ops, tiles, st)
                    : launch_fwd<256, OutT, 1, 64, AF>(job, ops, tiles, st);
    }
  }
  switch (job.tile_n) {
    case 64:
      if constexpr (!AF) return launch_fwd<64, OutT, 3, fwd_bk<64>()>(job, ops, tiles, st);
      return 1;
    case 128: return launch_fwd<128, OutT, 3, fwd_bk<128>(), AF>(job, ops, tiles, st);
    default: return launch_fwd<256, OutT, 3, fwd_bk<256>(), AF>(job, ops, tiles, st);
  }
}

}  // namespace

bool hgt_typed_linear_tc_supported(int64_t lda, int32_t K, int32_t cb_width) {
  (void)lda;
  return cb_width % 16 == 0 && cb_width > 0 && K >= BK;
}

// 64-column tiles read A split by k_split_bf16: each 128-row block of A is read by every column tile of its group (seven
// at d = 400), and splitting it once up front is cheaper than splitting it in every tile (DESIGN.md §4).
static bool splits_a_first(int32_t cb_width) { return pick_tile_n(cb_width) == 64; }

// W's halves (P = 1 needs no lo), A's halves for 64-column tiles, and the output maps.  At 128 / 256 columns A needs
// none: the GEMM splits fp32 A itself.  An fp32 A that TMA cannot load splits into stream-ordered memory of its own
// (tc_run).  The presplit entry points take the P = 3 size.
size_t hgt_typed_linear_tc_workspace(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K, int32_t cb_width,
                                     int32_t products) {
  int64_t a_rows, w_rows;
  extents(h_groups, n_groups, cb_width, &a_rows, &w_rows);
  const int Kp = (K + 7) / 8 * 8;
  const size_t halves = products == 1 ? 1 : 2;
  const size_t a = splits_a_first(cb_width) ? halves * hgt_align_up((size_t)a_rows * Kp * 2, 256) : 0;
  return 4 * 256 + a + halves * hgt_align_up((size_t)w_rows * Kp * 2, 256) +
         hgt_align_up((size_t)n_out_maps(h_groups, n_groups) * 2 * sizeof(CUtensorMap), 256);   // two for 24-bit tables
}

template <class OutT>
static int tc_run(const float* A, int64_t lda, const __nv_bfloat16* a_hi_in, const __nv_bfloat16* a_lo_in,
                  const float* W, const float* bias, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                  const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* cblocks, OutT* out,
                  int32_t products, void* workspace, size_t workspace_bytes, cudaStream_t st, float* out32 = nullptr,
                  int64_t t24_off = 0);

int hgt_typed_linear_tc(const float* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                        const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                        const hgt_lin_cblock* cblocks, float* out, int32_t products, void* workspace,
                        size_t workspace_bytes, cudaStream_t st) {
  return tc_run(A, lda, nullptr, nullptr, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, products,
                workspace, workspace_bytes, st);
}

int hgt_typed_linear_tc(const float* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                        const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                        const hgt_lin_cblock* cblocks, __nv_bfloat16* out, int32_t products, void* workspace,
                        size_t workspace_bytes, cudaStream_t st) {
  return tc_run(A, lda, nullptr, nullptr, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, products,
                workspace, workspace_bytes, st);
}

int hgt_typed_linear_tc(const float* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                        const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                        const hgt_lin_cblock* cblocks, float* out32, int64_t t24_off, hgt_t24* out,
                        int32_t products, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  return tc_run(A, lda, nullptr, nullptr, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, products,
                workspace, workspace_bytes, st, out32, t24_off);
}

int hgt_typed_linear_tc(const float* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                        const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                        const hgt_lin_cblock* cblocks, float* out32, int64_t t24_off, hgt_bs16* out,
                        int32_t products, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  return tc_run(A, lda, nullptr, nullptr, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, products,
                workspace, workspace_bytes, st, out32, t24_off);
}

extern "C" int hgt_typed_linear_presplit_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K,
                                                         int32_t cb_width, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && (h_groups || n_groups == 0), "hgt_typed_linear_presplit_workspace_bytes: NULL argument");
  *out_bytes = n_groups > 0 ? hgt_typed_linear_tc_workspace(h_groups, n_groups, K, cb_width, 3) : 0;   // fits P = 1 too
  return 0;
}

template <class OutT>
static int typed_linear_presplit(const void* a_hi, const void* a_lo, const float* W, const float* bias, int32_t K,
                                 int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                 int32_t n_groups, const hgt_lin_cblock* cblocks, OutT* out, void* workspace,
                                 size_t workspace_bytes, cudaStream_t st, float* out32 = nullptr,
                                 int64_t t24_off = 0) {
  HGT_REQUIRE(a_hi, "hgt_typed_linear_presplit: NULL operand");          // a_lo == NULL: one bf16 product
  HGT_REQUIRE(K % 8 == 0 && hgt_typed_linear_tc_supported(K, K, cb_width),
              "hgt_typed_linear_presplit: unsupported shape K=%d cb_width=%d", K, cb_width);
  if (n_groups == 0) return 0;
  if (n_groups > kMaxGroups) {                               // see hgt_typed_linear: chunked launches
    for (int g0 = 0; g0 < n_groups; g0 += kMaxGroups) {
      const int n = n_groups - g0 < kMaxGroups ? n_groups - g0 : kMaxGroups;
      int rc = typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups + g0, h_groups + g0, n, cblocks, out,
                                     workspace, workspace_bytes, st, out32, t24_off);
      if (rc) return rc;
    }
    return 0;
  }
  return tc_run(nullptr, 0, reinterpret_cast<const __nv_bfloat16*>(a_hi), reinterpret_cast<const __nv_bfloat16*>(a_lo),
                W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, a_lo ? 3 : 1, workspace, workspace_bytes,
                st, out32, t24_off);
}

extern "C" int hgt_typed_linear_presplit(const void* a_hi, const void* a_lo, const float* W, const float* bias,
                                         int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                         const hgt_lin_group* h_groups, int32_t n_groups,
                                         const hgt_lin_cblock* cblocks, float* out, void* workspace,
                                         size_t workspace_bytes, void* stream_) {
  return typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, workspace,
                               workspace_bytes, (cudaStream_t)stream_);
}

extern "C" int hgt_typed_linear_presplit_bf16(const void* a_hi, const void* a_lo, const float* W, const float* bias,
                                              int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                              const hgt_lin_group* h_groups, int32_t n_groups,
                                              const hgt_lin_cblock* cblocks, void* out, void* workspace,
                                              size_t workspace_bytes, void* stream_) {
  return typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks,
                               static_cast<__nv_bfloat16*>(out), workspace, workspace_bytes, (cudaStream_t)stream_);
}

extern "C" int hgt_typed_linear_presplit_t24(const void* a_hi, const void* a_lo, const float* W, const float* bias,
                                             int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                             const hgt_lin_group* h_groups, int32_t n_groups,
                                             const hgt_lin_cblock* cblocks, float* out, int64_t t24_off, void* out24,
                                             void* workspace, size_t workspace_bytes, void* stream_) {
  return typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks,
                               static_cast<hgt_t24*>(out24), workspace, workspace_bytes, (cudaStream_t)stream_, out,
                               t24_off);
}

extern "C" int hgt_typed_linear_presplit_bs16(const void* a_hi, const void* a_lo, const float* W, const float* bias,
                                              int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                              const hgt_lin_group* h_groups, int32_t n_groups,
                                              const hgt_lin_cblock* cblocks, float* out, int64_t t24_off, void* out16,
                                              void* workspace, size_t workspace_bytes, void* stream_) {
  HGT_REQUIRE(cb_width % 16 == 0, "hgt_typed_linear_presplit_bs16: needs cb_width %% 16 == 0 (cb_width=%d)", cb_width);
  return typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks,
                               static_cast<hgt_bs16*>(out16), workspace, workspace_bytes, (cudaStream_t)stream_, out,
                               t24_off);
}

template <class OutT>
static int tc_run(const float* A, int64_t lda, const __nv_bfloat16* a_hi_in, const __nv_bfloat16* a_lo_in,
                  const float* W, const float* bias, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                  const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* cblocks, OutT* out,
                  int32_t products, void* workspace, size_t workspace_bytes, cudaStream_t st, float* out32,
                  int64_t t24_off) {
  HGT_REQUIRE(hgt_typed_linear_tc_supported(lda, K, cb_width), "hgt_typed_linear(tc): unsupported K=%d cb_width=%d", K,
              cb_width);
  HGT_REQUIRE(products == 3 || products == 1, "hgt_typed_linear(tc): products=%d", products);
  const bool one = products == 1;
  FwdOps ops;
  ops.out32 = out32;
  ops.t24_off = t24_off;
  ops.K = K;
  ops.Kp = (K + 7) / 8 * 8;
  extents(h_groups, n_groups, cb_width, &ops.a_rows, &ops.w_rows);
  size_t need = hgt_typed_linear_tc_workspace(h_groups, n_groups, K, cb_width, products);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_typed_linear(tc): workspace too small (%zu < %zu)",
              workspace_bytes, need);
  const size_t w_half = hgt_align_up((size_t)ops.w_rows * ops.Kp * 2, 256);
  const size_t a_half = hgt_align_up((size_t)ops.a_rows * ops.Kp * 2, 256);
  char* p = reinterpret_cast<char*>(hgt_align_up(reinterpret_cast<size_t>(workspace), 256));
  __nv_bfloat16* a_ws = nullptr;                              // A's halves in the workspace (64-column tiles)
  if (splits_a_first(cb_width)) a_ws = reinterpret_cast<__nv_bfloat16*>(p), p += (one ? 1 : 2) * a_half;
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(p); p += w_half;
  __nv_bfloat16* w_lo = one ? nullptr : reinterpret_cast<__nv_bfloat16*>(p); p += one ? 0 : w_half;
  CUtensorMap* out_maps = reinterpret_cast<CUtensorMap*>(p);
  ops.w_hi = w_hi;
  ops.w_lo = w_lo;
  int64_t n = ops.w_rows * (ops.Kp / 4);
  if (n > 0) k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, K, ops.w_rows, K, ops.Kp, w_hi, w_lo);
  HGT_LAUNCH_CHECK();
  ops.a32 = A;
  ops.lda = lda;
  ops.a_hi = a_hi_in;                                         // split by the producer (e.g. the edge kernel)
  ops.a_lo = one ? nullptr : a_lo_in;
  if (a_hi_in)
    return run_fwd<OutT, false>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st);
  n = ops.a_rows * (ops.Kp / 4);
  if (a_ws) {
    if (n == 0) return 0;
    ops.a_hi = a_ws;
    ops.a_lo = one ? nullptr : a_ws + a_half / 2;
    k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, lda, ops.a_rows, K, ops.Kp, a_ws,
                                                              const_cast<__nv_bfloat16*>(ops.a_lo));
    HGT_LAUNCH_CHECK();
    return run_fwd<OutT, false>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st);
  }
  if (a_fp32_loadable(A, lda))                                // the GEMM splits A as it loads it
    return run_fwd<OutT, true>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st);
  // An fp32 A that TMA cannot load (base not 16-byte aligned, or lda % 4 != 0) is split first, into stream-ordered
  // memory of its own, so that the workspace need not hold halves of A for every caller.
  if (n == 0) return 0;
  void* halves = nullptr;
  HGT_CHECK_CUDA(cudaMallocAsync(&halves, (one ? 1 : 2) * a_half, st));
  const int rc = [&]() -> int {
    __nv_bfloat16* a_hi = static_cast<__nv_bfloat16*>(halves);
    __nv_bfloat16* a_lo = one ? nullptr : a_hi + a_half / 2;
    k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, lda, ops.a_rows, K, ops.Kp, a_hi, a_lo);
    HGT_LAUNCH_CHECK();
    ops.a_hi = a_hi;
    ops.a_lo = a_lo;
    return run_fwd<OutT, false>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st);
  }();
  const cudaError_t freed = cudaFreeAsync(halves, st);
  if (rc) return rc;
  HGT_CHECK_CUDA(freed);
  return 0;
}

// bf16 A (see the top of the file): W split as for fp32 A, A read in place or copied into zero-padded rows first.  The
// workspace is hgt_typed_linear_tc_workspace's for the same shape (the A halves it reserves for 64-column tiles stay
// unused).
int hgt_typed_linear_tc_bf16a(const __nv_bfloat16* A, int64_t lda, const float* W, const float* bias, int32_t K,
                              int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                              int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int32_t products,
                              void* workspace, size_t workspace_bytes, cudaStream_t st) {
  HGT_REQUIRE(hgt_typed_linear_tc_supported(lda, K, cb_width), "hgt_typed_linear_bf16a(tc): unsupported K=%d cb_width=%d",
              K, cb_width);
  HGT_REQUIRE(products == 3 || products == 1, "hgt_typed_linear_bf16a(tc): products=%d", products);
  const bool one = products == 1;
  FwdOps ops;
  ops.a32 = nullptr;
  ops.lda = 0;
  ops.out32 = nullptr;
  ops.t24_off = 0;
  ops.K = K;
  ops.Kp = (K + 7) / 8 * 8;
  extents(h_groups, n_groups, cb_width, &ops.a_rows, &ops.w_rows);
  const size_t need = hgt_typed_linear_tc_workspace(h_groups, n_groups, K, cb_width, products);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_typed_linear_bf16a(tc): workspace too small (%zu < %zu)",
              workspace_bytes, need);
  const size_t w_half = hgt_align_up((size_t)ops.w_rows * ops.Kp * 2, 256);
  const size_t a_pad = hgt_align_up((size_t)ops.a_rows * ops.Kp * 2, 256);
  char* p = reinterpret_cast<char*>(hgt_align_up(reinterpret_cast<size_t>(workspace), 256));
  if (splits_a_first(cb_width)) p += (one ? 1 : 2) * a_pad;
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(p); p += w_half;
  __nv_bfloat16* w_lo = one ? nullptr : reinterpret_cast<__nv_bfloat16*>(p); p += one ? 0 : w_half;
  CUtensorMap* out_maps = reinterpret_cast<CUtensorMap*>(p);
  ops.w_hi = w_hi;
  ops.w_lo = w_lo;
  int64_t n = ops.w_rows * (ops.Kp / 4);
  if (n > 0) k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, K, ops.w_rows, K, ops.Kp, w_hi, w_lo);
  HGT_LAUNCH_CHECK();
  ops.a_lo = nullptr;
  if (A && (reinterpret_cast<uintptr_t>(A) & 15) == 0 && lda % 8 == 0 && K % 8 == 0) {
    ops.a_hi = A;
    ops.a_ld = lda;
    return run_fwd<float, false>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st, true);
  }
  n = ops.a_rows * (ops.Kp / 4);
  if (n == 0) return 0;
  void* padded = nullptr;
  HGT_CHECK_CUDA(cudaMallocAsync(&padded, a_pad, st));
  const int rc = [&]() -> int {
    k_pad_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, lda, ops.a_rows, K, ops.Kp,
                                                            static_cast<__nv_bfloat16*>(padded));
    HGT_LAUNCH_CHECK();
    ops.a_hi = static_cast<const __nv_bfloat16*>(padded);
    return run_fwd<float, false>(ops, bias, cb_width, groups, h_groups, n_groups, cblocks, out, out_maps, one, st, true);
  }();
  const cudaError_t freed = cudaFreeAsync(padded, st);
  if (rc) return rc;
  HGT_CHECK_CUDA(freed);
  return 0;
}
