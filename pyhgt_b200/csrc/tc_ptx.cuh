// Hopper (sm_90a) tensor-core plumbing shared by the typed-linear GEMMs (linear_tc.cu forward, linear_bwd.cu dX / dW):
// mbarrier, TMA tile loads, wgmma shared-memory descriptors and instructions, and one warp-specialised kernel template.
//
// Every GEMM here is the split-bf16 x3 product: fp32 operands are split into x = x_hi + x_lo (two bf16 terms) and
//     A*B  ~=  A_hi*B_hi + A_hi*B_lo + A_lo*B_hi            (dropped term ~2^-18 relative)
// is accumulated in one fp32 register accumulator, three bf16 wgmma products per k-step.
//
// split3_tile<BN, MN, KB, Job>: the body of a persistent kernel (384 threads, at most one CTA per SM) whose CTAs walk the
// 128 x BN output tiles blockIdx.x, blockIdx.x + gridDim.x, ...
//   warpgroup 0   TMA producer (one thread): per k-block one pipeline stage {A_hi, A_lo, B_hi, B_lo}; the ring runs on
//                 across tiles, so the next tile's first stages load while the consumers finish and store this one
//   warpgroups 1-2  consumers: rows [64 c, 64 c + 64) of the tile, wgmma m64nBNk16 from shared memory
// Operand tiles are TMA boxes with SWIZZLE_128B, 64 bf16 (128 bytes) along the inner dimension (KB = 64), or with
// SWIZZLE_64B, 32 bf16 (KB = 32: half the stage, twice the ring depth).  MN = false: both operands K-major (inner dimension =
// reduction); MN = true: both MN-major (inner dimension = output row / column, the reduction runs over the box rows; KB = 64
// only).  The Job supplies the tile decode, the loads of one stage and the epilogue.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "common.cuh"

namespace tcp {

__device__ __forceinline__ uint32_t s_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// sm_90 shared-memory matrix descriptor, SWIZZLE_128B (KB = 64, layout type 1 at bits 62-63) or SWIZZLE_64B (KB = 32,
// layout type 2).  Tiles start 1024-byte aligned (base offset 0).  K-major: rows of 2 * KB bytes, 8-row swizzle atoms
// SBO = 16 * KB bytes apart, LBO unused.  MN-major (KB = 64): 64 MN-elements per 128-byte row, one row per k; groups of 8
// k-rows SBO = 1024 bytes apart, 64-element MN atoms LBO apart.
template <int KB>
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
  static_assert(KB == 64 || KB == 32, "k-block of 64 (SWIZZLE_128B) or 32 (SWIZZLE_64B) bf16");
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((16 * KB) >> 4) << 32;
  d |= (uint64_t)(KB == 64 ? 1 : 2) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] += A[64 x 16] * B[16 x N]; TA / TB = 1 selects an MN-major operand.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}

constexpr int BM = 128;                           // tile rows: two consumer warpgroups of 64
constexpr int BK = 64;                            // 64 bf16 = 128 bytes = one SWIZZLE_128B row
constexpr int TILE_THREADS = 384;
constexpr uint32_t A_BYTES = BM * BK * 2;         // one A operand (hi or lo) of a stage: 16 KB
constexpr uint32_t ATOM_BYTES = 64 * BK * 2;      // one {64 x 64} bf16 box: 8 KB
constexpr uint32_t SMEM_BUDGET = 192 * 1024;      // pipeline stages; H100 allows 227 KB of shared memory per block
constexpr uint32_t OUT_STAGE_BYTES = 2 * 64 * 64 * 4;  // epilogue staging after the ring: one 64 x 64 fp32 block per consumer

// Stage layout for a k-block of KB bf16: {A_hi, A_lo, B_hi, B_lo}; a consumer's 64-row A slab is one atom.
template <int KB> constexpr uint32_t a_bytes() { return BM * KB * 2; }
template <int KB> constexpr uint32_t atom_bytes() { return 64 * KB * 2; }
template <int BN, int KB = BK> constexpr uint32_t stage_bytes() { return 2 * a_bytes<KB>() + 2 * (uint32_t)BN * KB * 2; }
template <int BN, int KB = BK> constexpr int n_stages() { return (int)(SMEM_BUDGET / stage_bytes<BN, KB>()); }
template <int BN, int KB = BK> constexpr size_t tile_smem_bytes() {
  return 1024 + (size_t)n_stages<BN, KB>() * stage_bytes<BN, KB>() + OUT_STAGE_BYTES +
         2 * n_stages<BN, KB>() * sizeof(uint64_t);
}
static_assert(tile_smem_bytes<256, 32>() <= 227 * 1024 && tile_smem_bytes<256>() <= 227 * 1024 &&
                  tile_smem_bytes<128, 32>() <= 227 * 1024 && tile_smem_bytes<64>() <= 227 * 1024,
              "ring + epilogue staging must fit the 227 KB a block may use");

// Output tile width: 64, 128 or 256 columns, the one that pads `width` least (ties go to the wider tile).  Columns past
// `width` are computed on zero or neighbouring operands and masked in the epilogue.
inline int pick_tile_n(int64_t width) {
  int best = 64;
  int64_t best_pad = (width + 63) / 64 * 64;
  for (int bn : {128, 256}) {
    const int64_t pad = (width + bn - 1) / bn * bn;
    if (pad <= best_pad) best = bn, best_pad = pad;
  }
  return best;
}

// Grid of a split3_tile kernel: one CTA per SM (its shared memory leaves no room for a second), no more CTAs than tiles.
inline unsigned persistent_grid(int tiles) {
  const int sms = hgt_sm_count();
  return (unsigned)(tiles < sms ? tiles : sms);
}

// The 3 products of one k-block.  a_hi / a_lo: this warpgroup's 64-row A slab; b_hi / b_lo: the BN-column B tile.
template <int BN, bool MN, int KB>
__device__ __forceinline__ void mma_kblock(float* acc, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  static_assert(!MN || KB == 64, "MN-major operands use 64-row k-blocks");
  constexpr uint32_t kstep = MN ? 16 * 128 : 32;       // 16 k: 16 rows of 128 bytes, or 32 bytes inside the swizzle row
  constexpr uint32_t lbo = MN ? ATOM_BYTES : 16;
  constexpr uint32_t b_half = 128 * KB * 2;            // columns 128-255 of B: 128 rows (K-major) or two 64-column atoms
  constexpr int T = MN ? 1 : 0;
#pragma unroll
  for (int k = 0; k < KB / 16; ++k) {
    const uint32_t o = (uint32_t)k * kstep;
    const uint64_t ah = make_desc<KB>(a_hi + o, lbo), al = make_desc<KB>(a_lo + o, lbo);
    const uint64_t bh = make_desc<KB>(b_hi + o, lbo), bl = make_desc<KB>(b_lo + o, lbo);
    if constexpr (BN == 64) {
      wgmma_n64<T, T>(acc, ah, bh);
      wgmma_n64<T, T>(acc, ah, bl);
      wgmma_n64<T, T>(acc, al, bh);
    } else {
      wgmma_n128<T, T>(acc, ah, bh);
      wgmma_n128<T, T>(acc, ah, bl);
      wgmma_n128<T, T>(acc, al, bh);
      if constexpr (BN == 256) {
        const uint64_t bh2 = make_desc<KB>(b_hi + o + b_half, lbo), bl2 = make_desc<KB>(b_lo + o + b_half, lbo);
        wgmma_n128<T, T>(acc + 64, ah, bh2);
        wgmma_n128<T, T>(acc + 64, ah, bl2);
        wgmma_n128<T, T>(acc + 64, al, bh2);
      }
    }
  }
}

// Accumulator fragment of wgmma m64nN (f32): acc[4 j + 2 h + e] is row 16 * warp + lane / 4 + 8 h of the warpgroup's 64
// rows, column 8 j + 2 (lane % 4) + e.  `fn(row, col, v0, v1)` gets each pair of neighbouring columns.
template <int BN, class Fn>
__device__ __forceinline__ void for_each_pair(const float* acc, int wq, int lane, Fn fn) {
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    fn(r0, 8 * j + c0, acc[4 * j], acc[4 * j + 1]);
    fn(r0 + 8, 8 * j + c0, acc[4 * j + 2], acc[4 * j + 3]);
  }
}

__device__ __forceinline__ void bar_sync_named(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Coalesced epilogue of one consumer warpgroup (c): its 64 x BN accumulator goes out in 64-column blocks through `stage`
// (64 x 64 fp32; 16-byte chunk q of row r sits at chunk q ^ 2 (r & 7), which keeps both the fragment writes and the row
// reads free of bank conflicts).  Each row of a block is then read by 16 consecutive threads, so a warp writes two whole
// 256-byte row segments per instruction instead of 32-byte pieces of eight rows.
// pair(row, col, v0, v1) -> float2 gives the values of two neighbouring columns (e.g. with the bias added);
// write(row, col, float4) stores columns col .. col + 3 of a row.
template <int BN, class Pair, class Write>
__device__ __forceinline__ void store_staged(const float* acc, float* stage, int c, int wq, int lane, Pair pair,
                                             Write write) {
  const int tid = 32 * wq + lane, r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int blk = 0; blk < BN / 64; ++blk) {
    bar_sync_named(1 + c, 128);                                 // the previous block has been read out
#pragma unroll
    for (int j = 8 * blk; j < 8 * blk + 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h, lc = 8 * j + c0 - 64 * blk;
        const float2 v = pair(r, 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        *reinterpret_cast<float2*>(stage + r * 64 + (((lc >> 2) ^ ((r & 7) << 1)) << 2) + (lc & 3)) = v;
      }
    }
    bar_sync_named(1 + c, 128);
    const int q = tid & 15;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = (tid >> 4) + 8 * i;
      write(r, 64 * blk + 4 * q, *reinterpret_cast<const float4*>(stage + r * 64 + ((q ^ ((r & 7) << 1)) << 2)));
    }
  }
}

// Called by a __global__ kernel with __launch_bounds__(TILE_THREADS, 1) and tile_smem_bytes<BN, KB>() of dynamic shared
// memory; `job` is the kernel's __grid_constant__ parameter (it holds the tensor maps), `n_tiles` the number of tiles
// job.decode() accepts.  Every tile's k-blocks run in ascending order into a freshly zeroed accumulator, so a tile's
// result does not depend on the grid size or on which CTA computes it.
template <int BN, bool MN, int KB, class Job>
__device__ __forceinline__ void split3_tile(const Job& job, int n_tiles) {
  constexpr int S = n_stages<BN, KB>();
  constexpr uint32_t STAGE = stage_bytes<BN, KB>();
  constexpr uint32_t A = a_bytes<KB>(), ATOM = atom_bytes<KB>();
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (s_u32(smem_dyn) & 1023u)) & 1023u);
  float* out_stage = reinterpret_cast<float*>(smem + (size_t)S * STAGE);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)S * STAGE + OUT_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + S;
  const uint32_t base = s_u32(smem);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(s_u32(&full_bar[s]), 1);
      mbar_init(s_u32(&empty_bar[s]), 8);                          // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Ring position shared by all tiles of this CTA: stage s, and the parity of its current use.
  int s = 0;
  uint32_t phase = 0;
  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x == 0) {
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        typename Job::Tile t;
        const int iters = job.decode(tile, t);
        job.prefetch(t);
        for (int it = 0; it < iters; ++it) {
          mbar_wait(s_u32(&empty_bar[s]), phase ^ 1u);
          const uint32_t bar = s_u32(&full_bar[s]);
          mbar_expect_tx(bar, STAGE);
          job.template load<BN>(t, it, base + (uint32_t)s * STAGE, bar);
          if (++s == S) s = 0, phase ^= 1u;
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int c = wg - 1;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      typename Job::Tile t;
      const int iters = job.decode(tile, t);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = 0;                                               // stage of the previous k-block
      for (int it = 0; it < iters; ++it) {
        mbar_wait(s_u32(&full_bar[s]), phase);
        const uint32_t sa = base + (uint32_t)s * STAGE;
        wgmma_fence();
        mma_kblock<BN, MN, KB>(acc, sa + c * ATOM, sa + A + c * ATOM, sa + 2 * A, sa + 2 * A + (uint32_t)BN * KB * 2);
        wgmma_commit();
        if (it > 0) {                                             // the previous k-block's products have retired
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(s_u32(&empty_bar[prev]));
        }
        prev = s;
        if (++s == S) s = 0, phase ^= 1u;
      }
      wgmma_wait<0>();
      if (iters > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(s_u32(&empty_bar[prev]));     // the producer may refill it during the store
        job.template store<BN>(t, acc, out_stage + c * 64 * 64, c, warp & 3, lane);
      }
    }
  }
}

}  // namespace tcp
