// Hopper (sm_90a) tensor-core plumbing shared by the typed-linear GEMMs (linear_tc.cu forward, linear_bwd.cu dX / dW):
// mbarrier, TMA tile loads, wgmma shared-memory descriptors and instructions, and one warp-specialised kernel template.
//
// By default every GEMM here is the split-bf16 x3 product (P = 3): fp32 operands are split into x = x_hi + x_lo (two bf16
// terms) and
//     A*B  ~=  A_hi*B_hi + A_hi*B_lo + A_lo*B_hi            (dropped term ~2^-18 relative)
// is accumulated in one fp32 register accumulator, three bf16 wgmma products per k-step.  P = 1 is the single bf16
// product A_hi*B_hi (torch.set_float32_matmul_precision("medium")): a stage holds {A_hi, B_hi} only, so it is half the
// size and the ring twice as deep.  P = 2 and P = 4 are the x3 product with one operand exact in bf16 (its lo half is
// zero, so the product with it adds exact zeros and is skipped): P = 2, A exact, runs A_hi*B_hi + A_hi*B_lo from
// {A_hi, B_hi, B_lo}; P = 4, B exact, runs A_hi*B_hi + A_lo*B_hi from {A_hi, A_lo, B_hi}.  The products that remain run
// in the order P = 3 runs them, so the accumulator takes the same values.
//
// split3_tile<BN, MN, KB, OUT, P, Job>: the body of a persistent kernel (384 threads, at most one CTA per SM) whose CTAs walk the
// 128 x BN output tiles blockIdx.x, blockIdx.x + gridDim.x, ...
//   warpgroup 0   TMA producer (one thread): per k-block one pipeline stage {A_hi, A_lo, B_hi, B_lo} (P = 3) or
//                 {A_hi, B_hi} (P = 1); the ring runs on
//                 across tiles, so the next tile's first stages load while the consumers finish and store this one
//   warpgroups 1-2  consumers: rows [64 c, 64 c + 64) of the tile, wgmma m64nBNk16 from shared memory
// AF = true (the forward's fp32 A): a stage holds A as fp32 in place of its halves, and each consumer splits its rows
// into hi / lo in shared memory (split_a_slab) before the k-block's products.
// Operand tiles are TMA boxes with SWIZZLE_128B, 64 bf16 (128 bytes) along the inner dimension (KB = 64), or with
// SWIZZLE_64B, 32 bf16 (KB = 32: half the stage, twice the ring depth).  MN = false: both operands K-major (inner dimension =
// reduction); MN = true: both MN-major (inner dimension = output row / column, the reduction runs over the box rows; KB = 64
// only).  The Job supplies the tile decode, the loads of one stage and the epilogue (store_staged: st.global from a shared
// staging block; store_tma: TMA tensor stores that drain while the consumer runs the next tile).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include <type_traits>

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
// SBO bytes apart (16 * KB when packed), LBO unused.  MN-major (KB = 64): 64 MN-elements per 128-byte row, one row per k;
// groups of 8 k-rows SBO = 1024 bytes apart, 64-element MN atoms LBO apart.
template <int KB>
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes = 16 * KB) {
  static_assert(KB == 64 || KB == 32, "k-block of 64 (SWIZZLE_128B) or 32 (SWIZZLE_64B) bf16");
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
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
constexpr uint32_t SMEM_LIMIT = 227 * 1024;       // shared memory a block may use on H100
constexpr uint32_t SMEM_BUDGET = 192 * 1024;      // most the pipeline stages take
constexpr uint32_t OUT_STAGE_BYTES = 2 * 64 * 64 * 4;  // epilogue staging after the ring: one 64 x 64 fp32 block per consumer
// Staging of the tensor-store epilogue (store_tma): per consumer two 64 x 64 buffers (at most fp32), so one buffer fills
// while the other drains.
constexpr uint32_t TMA_BUF_BYTES = 64 * 64 * 4;
constexpr uint32_t TMA_STAGE_BYTES = 2 * 2 * TMA_BUF_BYTES;

// Stage layout for a k-block of KB bf16: {A_hi, A_lo, B_hi, B_lo} at P = 3, {A_hi, B_hi} at P = 1; a consumer's 64-row A
// slab is one atom, B_lo follows B_hi.  AF (fp32 A): the A part is the k-block of A as fp32, KB / 32 boxes of 128 rows x
// 32 floats (A32_BOX bytes each), which the consumers split in place (split_a_slab); at P = 3 that is the size of
// {A_hi, A_lo}, at P = 1 twice that of A_hi.  The ring takes what the epilogue staging (OUT bytes) and the barriers leave,
// up to SMEM_BUDGET.
constexpr uint32_t A32_BOX = BM * 32 * 4;         // one fp32 A box: 128 rows x 128 bytes, 16 KB
template <int KB> constexpr uint32_t a_bytes() { return BM * KB * 2; }
template <int KB> constexpr uint32_t atom_bytes() { return 64 * KB * 2; }
// Which lo halves a product count P loads and multiplies.
template <int P> constexpr bool has_a_lo() { return P == 3 || P == 4; }
template <int P> constexpr bool has_b_lo() { return P == 3 || P == 2; }
template <int KB, int P, bool AF = false> constexpr uint32_t b_offset() {                 // B_hi in a stage
  return AF ? 2u * a_bytes<KB>() : (has_a_lo<P>() ? 2u : 1u) * a_bytes<KB>();
}
template <int BN, int KB = BK, int P = 3, bool AF = false> constexpr uint32_t stage_bytes() {
  static_assert(P == 3 || P == 1 || ((P == 2 || P == 4) && !AF), "split (3), hi only (1), one exact operand (2, 4)");
  return b_offset<KB, P, AF>() + (has_b_lo<P>() ? 2u : 1u) * (uint32_t)BN * KB * 2;
}
template <int BN, int KB = BK, uint32_t OUT = OUT_STAGE_BYTES, int P = 3, bool AF = false> constexpr int n_stages() {
  constexpr uint32_t left = SMEM_LIMIT - 1024 - OUT - 256;
  return (int)((left < SMEM_BUDGET ? left : SMEM_BUDGET) / stage_bytes<BN, KB, P, AF>());
}
template <int BN, int KB = BK, uint32_t OUT = OUT_STAGE_BYTES, int P = 3, bool AF = false>
constexpr size_t tile_smem_bytes() {
  return 1024 + (size_t)n_stages<BN, KB, OUT, P, AF>() * stage_bytes<BN, KB, P, AF>() + OUT +
         2 * n_stages<BN, KB, OUT, P, AF>() * sizeof(uint64_t);
}
// Every forward (AF and presplit) and backward instance.
template <bool AF> constexpr bool fwd_fits() {
  return tile_smem_bytes<256, 32, TMA_STAGE_BYTES, 3, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<128, 32, TMA_STAGE_BYTES, 3, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<64, 64, OUT_STAGE_BYTES, 3, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<256, 32, TMA_STAGE_BYTES, 1, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<256, 64, TMA_STAGE_BYTES, 1, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<128, 32, TMA_STAGE_BYTES, 1, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<128, 64, TMA_STAGE_BYTES, 1, AF>() <= SMEM_LIMIT &&
         tile_smem_bytes<64, 64, OUT_STAGE_BYTES, 1, AF>() <= SMEM_LIMIT &&
         n_stages<256, 64, TMA_STAGE_BYTES, 1, AF>() >= 2 && n_stages<64, 64, OUT_STAGE_BYTES, 3, AF>() >= 2;
}
static_assert(fwd_fits<false>() && fwd_fits<true>() && tile_smem_bytes<256>() <= SMEM_LIMIT &&
                  tile_smem_bytes<256, 64, OUT_STAGE_BYTES, 1>() <= SMEM_LIMIT &&
                  tile_smem_bytes<128, 64, OUT_STAGE_BYTES, 1>() <= SMEM_LIMIT,
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

// The P products of one k-block.  a_hi / a_lo: this warpgroup's 64-row A slab, 8-row groups A_SBO bytes apart; b_hi /
// b_lo: the BN-column B tile (a lo half is not read where P has none: has_a_lo / has_b_lo).
template <int BN, bool MN, int KB, int P = 3, uint32_t A_SBO = 16 * KB>
__device__ __forceinline__ void mma_kblock(float* acc, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  static_assert(!MN || KB == 64, "MN-major operands use 64-row k-blocks");
  constexpr uint32_t kstep = MN ? 16 * 128 : 32;       // 16 k: 16 rows of 128 bytes, or 32 bytes inside the swizzle row
  constexpr uint32_t lbo = MN ? ATOM_BYTES : 16;
  constexpr uint32_t b_half = 128 * KB * 2;            // columns 128-255 of B: 128 rows (K-major) or two 64-column atoms
  constexpr int T = MN ? 1 : 0;
#pragma unroll
  for (int k = 0; k < KB / 16; ++k) {
    const uint32_t o = (uint32_t)k * kstep;
    const uint64_t ah = make_desc<KB>(a_hi + o, lbo, A_SBO), al = make_desc<KB>(a_lo + o, lbo, A_SBO);
    const uint64_t bh = make_desc<KB>(b_hi + o, lbo), bl = make_desc<KB>(b_lo + o, lbo);
    if constexpr (BN == 64) {
      wgmma_n64<T, T>(acc, ah, bh);
      if constexpr (has_b_lo<P>()) wgmma_n64<T, T>(acc, ah, bl);
      if constexpr (has_a_lo<P>()) wgmma_n64<T, T>(acc, al, bh);
    } else {
      wgmma_n128<T, T>(acc, ah, bh);
      if constexpr (has_b_lo<P>()) wgmma_n128<T, T>(acc, ah, bl);
      if constexpr (has_a_lo<P>()) wgmma_n128<T, T>(acc, al, bh);
      if constexpr (BN == 256) {
        const uint64_t bh2 = make_desc<KB>(b_hi + o + b_half, lbo), bl2 = make_desc<KB>(b_lo + o + b_half, lbo);
        wgmma_n128<T, T>(acc + 64, ah, bh2);
        if constexpr (has_b_lo<P>()) wgmma_n128<T, T>(acc + 64, ah, bl2);
        if constexpr (has_a_lo<P>()) wgmma_n128<T, T>(acc + 64, al, bh2);
      }
    }
  }
}

__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts64(uint32_t a, __nv_bfloat162 x, __nv_bfloat162 y) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(*reinterpret_cast<uint32_t*>(&x)),
               "r"(*reinterpret_cast<uint32_t*>(&y)) : "memory");
}

// AF: one consumer warpgroup splits its 64-row slab of a stage's fp32 A in place into the bf16 halves mma_kblock reads,
// x = hi + lo with hi = rn(x), lo = rn(x - hi), bitwise what k_split_bf16 writes.  `slab` is the slab in box 0 (box j,
// k 32 j .. 32 j + 31, lies A32_BOX * j further; 128-byte rows, 16-byte chunk q of row r at q ^ (r & 7), as TMA's
// SWIZZLE_128B writes it).  The halves are K-major:
//   KB = 32 (SWIZZLE_64B)  A_hi's 8-row groups 1024 bytes apart at the slab, A_lo 512 bytes after each group of A_hi;
//   KB = 64 (SWIZZLE_128B) A_hi packed at the slab, A_lo packed at the slab of box 1.
// Either way rows 16 w .. 16 w + 15 go where warp w read them from, so a warp only waits for itself between its loads and
// its stores.  A load takes four rows whose 64-bit stores are free of bank conflicts in each half-warp: rows {0, 1, 2, 3}
// + 4 i at KB = 32, {0, 4, 1, 5} (+ 2, + 8) at KB = 64.  The caller fences the stores to the async proxy and syncs the
// warpgroup before the products.
template <int KB>
__device__ __forceinline__ int split_row(int i, int lr) {
  return KB == 32 ? 4 * i + lr : 8 * (i >> 1) + 2 * (i & 1) + 4 * (lr & 1) + (lr >> 1);
}
template <int KB, int P>
__device__ __forceinline__ void split_a_slab(uint32_t slab, int wq, int lane) {
  constexpr int NB = KB / 32;
  const int lr = lane >> 3, q = lane & 7;
  float4 v[NB][4];
#pragma unroll
  for (int j = 0; j < NB; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i)
      v[j][i] = lds128(slab + j * A32_BOX + (16 * wq + split_row<KB>(i, lr)) * 128 + 16 * q);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < NB; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = 16 * wq + split_row<KB>(i, lr), x = r & 7;
      const int L = q ^ x;                                      // columns 32 j + 4 L .. + 3 of the k-block
      // two elements per conversion (cvt.rn.bf16x2.f32): the same round-to-nearest-even as __float2bfloat16_rn
      const float4 f = v[j][i];
      const __nv_bfloat162 h01 = __floats2bfloat162_rn(f.x, f.y), h23 = __floats2bfloat162_rn(f.z, f.w);
      const uint32_t half = (uint32_t)(L & 1) << 3;
      const uint32_t off = KB == 32 ? (r >> 3) * 1024 + x * 64 + ((((L >> 1) ^ (x >> 1)) << 4) | half)
                                    : (r >> 3) * 1024 + x * 128 + ((((4 * j + (L >> 1)) ^ x) << 4) | half);
      sts64(slab + off, h01, h23);
      if constexpr (P == 3) {
        const __nv_bfloat162 l01 = __floats2bfloat162_rn(f.x - __low2float(h01), f.y - __high2float(h01));
        const __nv_bfloat162 l23 = __floats2bfloat162_rn(f.z - __low2float(h23), f.w - __high2float(h23));
        sts64(slab + off + (KB == 32 ? 512 : A32_BOX), l01, l23);
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

// TMA tensor stores shared -> global (the async proxy).  Each thread tracks its own bulk groups.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(smem_src), "r"(c0), "r"(c1) : "memory");
}
// A tensor map written to global memory by an earlier kernel (generic proxy): acquire it for the TMA proxy.
__device__ __forceinline__ void tensormap_acquire(const CUtensorMap* m) {
  asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(m) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void put2(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }
__device__ __forceinline__ void put2(__nv_bfloat16* p, float2 v) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v.x, v.y);
}

// Two neighbouring 24-bit elements (hgt_t24_round of v.x, v.y): their hi halves as one u32 and their lo bytes as the low
// 16 bits of `lo` (the upper 16 are not defined).
__device__ __forceinline__ void t24_pair(float2 v, uint32_t& hi, uint32_t& lo) {
  const uint32_t a = hgt_t24_round(__float_as_uint(v.x)), b = hgt_t24_round(__float_as_uint(v.y));
  hi = __byte_perm(a, b, 0x7632);
  lo = __byte_perm(a, b, 0x0051);
}

template <class OutT> constexpr bool is_t24() { return std::is_same<OutT, hgt_t24>::value; }
template <class OutT> constexpr bool is_bs16() { return std::is_same<OutT, hgt_bs16>::value; }
// Gather-table outputs (24-bit or bs16): planar byte formats whose jobs write their fp32 column blocks elsewhere.
template <class OutT> constexpr bool is_table() { return is_t24<OutT>() || is_bs16<OutT>(); }
// Output tensor maps per (group, column block): one, or a hi-plane and a lo-plane map for 24-bit tables, a mantissa and
// a scale map for bs16 tables.
template <class OutT> constexpr int out_maps_per_block() { return is_table<OutT>() ? 2 : 1; }

// Asynchronous epilogue of one consumer warpgroup (c): its 64 x BN accumulator goes out in 64-column blocks.  Each block
// is written to shared memory as OutT in the SWIZZLE_128B layout of `map`'s boxes (128-byte rows, 64 rows; 16-byte chunk q
// of row r at q ^ (r & 7); fp32: two boxes of 32 columns, bf16: one box of 64) and sent to global memory by TMA tensor
// stores that one thread (the warpgroup's first) issues.  24-bit tables (hgt_t24): the hi halves as a bf16-like box of
// 64 u16 at the buffer and the lo bytes as a box of 64 u8 (64-byte rows, SWIZZLE_64B: chunk q of row r at
// q ^ ((r >> 1) & 3)) 8 KB further, stored through map[0] and map[1].  bs16 tables (hgt_bs16): the int16 mantissas as
// a bf16-like box of 64 through map[0]; the quad that holds a row's 16-column block finds its largest |x| with two
// shuffles, and lane h of the quad (rows r0 and r0 + 8 are h = 0 and 1) writes the row's four scales of the block into
// the tile's scale box (64 rows x BN / 16 bf16, unswizzled, in the unused upper half of buffer 0), which goes out
// through map[1] with the last block.  A block's own four scales per row are 8 bytes, below TMA's 16-byte inner box;
// scattered 8-byte st.global of them cost as much as the rest of the epilogue.  Before block 0 writes scales the
// previous tile's scale box has been read out (wait for all groups rather than all but the last).  The map's extents
// clip the rows past the group and the columns past the column block.  The stores drain while the consumer goes on to
// the next block or the next tile's products.
// Block b uses buffer b & 1 of `stage` (two TMA_BUF_BYTES buffers, 1024-byte aligned); BN / 64 is even, so the buffers
// alternate across tiles too.  Before a buffer is rewritten the issuing thread waits until the bulk group that read it two
// blocks earlier is done (it commits one group per block).
// pair(row, col, v0, v1) -> float2 as in store_staged; the block's row 0, column 0 is element (col0 + 64 b, row0) of
// the map; `cols`: columns of the tile inside the column block.
template <int BN, class OutT, class Pair>
__device__ __forceinline__ void store_tma(const float* acc, unsigned char* stage, int c, int wq, int lane, Pair pair,
                                          const CUtensorMap* map, int col0, int row0, int cols) {
  static_assert(BN % 128 == 0, "the two buffers alternate across tiles only for an even number of 64-column blocks");
  constexpr bool T24 = is_t24<OutT>(), BS16 = is_bs16<OutT>();
  constexpr int BOX_COLS = T24 || BS16 ? 64 : 128 / (int)sizeof(OutT);
  const bool issuer = wq == 0 && lane == 0;
  const int r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
  if (issuer) {
    tensormap_acquire(map);
    if constexpr (T24 || BS16) tensormap_acquire(map + 1);
  }
  unsigned char* const scale_box = stage + 8192;                 // bs16: 64 rows x BN / 8 bytes
#pragma unroll
  for (int blk = 0; blk < BN / 64; ++blk) {
    unsigned char* buf = stage + (blk & 1) * TMA_BUF_BYTES;
    if (issuer) {
      if (BS16 && blk == 0) bulk_wait_read<0>();                // ... and the previous tile's scale box
      else bulk_wait_read<1>();
    }
    bar_sync_named(1 + c, 128);                                 // the buffer has been read out
    if constexpr (BS16) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        uint32_t sc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {                           // 16-column block k: fragment columns j = 2k, 2k + 1
          const int j = 8 * blk + 2 * k;
          const float2 v0 = pair(r, 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          const float2 v1 = pair(r, 8 * j + 8 + c0, acc[4 * j + 4 + 2 * h], acc[4 * j + 4 + 2 * h + 1]);
          const uint32_t a = hgt_bs16_quad_amax(max(max(hgt_abs_bits(v0.x), hgt_abs_bits(v0.y)),
                                                    max(hgt_abs_bits(v1.x), hgt_abs_bits(v1.y))));
          float rc;
          sc[k] = hgt_bs16_scale(a, rc);
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float2 v = u ? v1 : v0;
            const uint32_t x = (uint32_t)(16 * k + 8 * u + c0) * 2;
            *reinterpret_cast<uint32_t*>(buf + r * 128 + ((((x >> 4) ^ (r & 7)) << 4) | (x & 15))) =
                hgt_bs16_pack(v.x, v.y, rc, sc[k]);
          }
        }
        if ((lane & 3) == h)
          *reinterpret_cast<uint2*>(scale_box + r * (BN / 8) + 8 * blk) =
              make_uint2(sc[0] | (sc[1] << 16), sc[2] | (sc[3] << 16));
      }
    } else {
#pragma unroll
      for (int j = 8 * blk; j < 8 * blk + 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 8 * h, lc = 8 * j + c0 - 64 * blk;
          const float2 v = pair(r, 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          if constexpr (T24) {
            uint32_t hi, lo;
            t24_pair(v, hi, lo);
            const uint32_t x = (uint32_t)lc * 2;
            *reinterpret_cast<uint32_t*>(buf + r * 128 + ((((x >> 4) ^ (r & 7)) << 4) | (x & 15))) = hi;
            *reinterpret_cast<uint16_t*>(buf + 8192 + r * 64 + ((((lc >> 4) ^ ((r >> 1) & 3)) << 4) | (lc & 15))) =
                (uint16_t)lo;
          } else {
            const uint32_t x = (uint32_t)(lc % BOX_COLS) * sizeof(OutT);     // byte in the box row
            put2(reinterpret_cast<OutT*>(buf + (lc / BOX_COLS) * 8192 + r * 128 + ((((x >> 4) ^ (r & 7)) << 4) | (x & 15))),
                 v);
          }
        }
      }
    }
    fence_proxy_async_smem();                                   // the writes are visible to the tensor stores
    bar_sync_named(1 + c, 128);
    if (issuer) {
#pragma unroll
      for (int bx = 0; bx < 64 / BOX_COLS; ++bx)
        if (64 * blk + BOX_COLS * bx < cols) tma_store_2d(map, s_u32(buf + bx * 8192), col0 + 64 * blk + BOX_COLS * bx, row0);
      if constexpr (T24)
        if (64 * blk < cols) tma_store_2d(map + 1, s_u32(buf + 8192), col0 + 64 * blk, row0);
      if constexpr (BS16)
        if (blk == BN / 64 - 1) tma_store_2d(map + 1, s_u32(scale_box), col0 / 16, row0);
      bulk_commit();
    }
  }
}

// Called by a __global__ kernel with __launch_bounds__(TILE_THREADS, 1) and tile_smem_bytes<BN, KB, OUT, P>() of dynamic shared
// memory; `job` is the kernel's __grid_constant__ parameter (it holds the tensor maps), `n_tiles` the number of tiles
// job.decode() accepts.  Every tile's k-blocks run in ascending order into a freshly zeroed accumulator, so a tile's
// result does not depend on the grid size or on which CTA computes it.  job.store gets consumer c's half of the OUT bytes
// of epilogue staging.  job.load<BN, KB, P>() fills one stage in the layout of stage_bytes<BN, KB, P, AF>().  AF: the stage
// holds A as fp32 (K-major only), and each consumer splits its slab of it (split_a_slab) before the k-block's products.
template <int BN, bool MN, int KB, uint32_t OUT = OUT_STAGE_BYTES, int P = 3, bool AF = false, class Job>
__device__ __forceinline__ void split3_tile(const Job& job, int n_tiles) {
  static_assert(!AF || !MN, "fp32 A is loaded K-major");
  constexpr int S = n_stages<BN, KB, OUT, P, AF>();
  constexpr uint32_t STAGE = stage_bytes<BN, KB, P, AF>();
  constexpr uint32_t ATOM = atom_bytes<KB>(), B = b_offset<KB, P, AF>();
  // A_lo of consumer 0 relative to its A_hi, and the stride of A's 8-row groups (split_a_slab's layout under AF)
  constexpr uint32_t A = AF ? (KB == 32 ? 512u : A32_BOX) : a_bytes<KB>();
  constexpr uint32_t A_SBO = AF ? 1024u : 16u * KB;
  constexpr uint32_t SLAB = AF ? 64u * 128u : ATOM;               // consumer c's A slab starts c * SLAB into the stage
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (s_u32(smem_dyn) & 1023u)) & 1023u);
  unsigned char* out_stage = smem + (size_t)S * STAGE;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)S * STAGE + OUT);
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
          job.template load<BN, KB, P>(t, it, base + (uint32_t)s * STAGE, bar);
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
        if constexpr (AF) {
          split_a_slab<KB, P>(sa + c * SLAB, warp & 3, lane);
          fence_proxy_async_smem();                               // the halves are visible to wgmma
          bar_sync_named(1 + c, 128);
        }
        wgmma_fence();
        mma_kblock<BN, MN, KB, P, A_SBO>(acc, sa + c * SLAB, sa + A + c * SLAB, sa + B, sa + B + (uint32_t)BN * KB * 2);
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
        job.template store<BN>(t, acc, reinterpret_cast<float*>(out_stage + c * (OUT / 2)), c, warp & 3, lane);
      }
    }
    bulk_wait_all();                                              // bulk stores of the epilogue, if it issued any
  }
}

}  // namespace tcp
