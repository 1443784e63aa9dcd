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
// wide (SWIZZLE_64B): at BN = 256 that makes a 4-deep ring of 48 KB stages instead of 2 x 96 KB.  BN = 64 keeps 64-wide
// k-blocks (SWIZZLE_128B, 4 stages): its k-blocks are short enough that halving them costs more in barrier waits than the
// deeper ring gains (measured on the d = 400 OAG shape).  Output tiles follow the same group / column-block tables
// as the SIMT kernel in linear.cu.
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

using namespace tcp;

constexpr int kMaxGroups = 64;
template <int BN> constexpr int fwd_bk() { return BN == 64 ? 64 : 32; }    // k-block of the forward GEMM

// ---- fp32 -> (bf16 hi, bf16 lo) split ------------------------------------------------------------
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
  *reinterpret_cast<uint2*>(lo + r * Kp + c) = *reinterpret_cast<uint2*>(l);
}

// ---- the GEMM: out_cb[m, n] = A[a_row0 + m, :] . W[w_row0 + cb * cb_width + n, :] (+ bias) ------------------------------
// Rows of a tile past the group and columns past the column block are computed on neighbouring (or zero-filled) operand
// rows and not stored.
struct FwdJob {
  CUtensorMap a_hi, a_lo, w_hi, w_lo;      // A box {fwd_bk, 128 rows}, W box {fwd_bk, tile_n rows}
  const float* bias;
  const hgt_lin_group* groups;
  const hgt_lin_cblock* cblocks;
  float* out;
  int n_groups, cb_width, k_blocks, tile_n, n_tiles_n;
  int32_t first_tile[kMaxGroups + 1];

  struct Tile {
    int a_row, w_row, cols;
    int64_t rows, ld;
    float* out;
    const float* bias;
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
    t.out = out + cblk.out_off + m0 * cblk.ld + n0;
    t.bias = (grp.has_bias && bias) ? bias + t.w_row : nullptr;
    return k_blocks;
  }
  __device__ void prefetch(const Tile&) const {
    prefetch_map(&a_hi); prefetch_map(&a_lo); prefetch_map(&w_hi); prefetch_map(&w_lo);
  }
  template <int BN>
  __device__ void load(const Tile& t, int kb, uint32_t sa, uint32_t bar) const {
    constexpr int KB = fwd_bk<BN>();
    constexpr uint32_t A = a_bytes<KB>();
    const int k = kb * KB;
    tma_load_2d(sa, &a_hi, k, t.a_row, bar);
    tma_load_2d(sa + A, &a_lo, k, t.a_row, bar);
    tma_load_2d(sa + 2 * A, &w_hi, k, t.w_row, bar);
    tma_load_2d(sa + 2 * A + BN * KB * 2, &w_lo, k, t.w_row, bar);
  }
  // Through shared memory, whole row segments per warp (tcp::store_staged).  cols is a multiple of 16, so a 4-column
  // group is either inside the column block or past it.
  template <int BN>
  __device__ void store(const Tile& t, const float* acc, float* stage, int c, int wq, int lane) const {
    float* o = t.out + (int64_t)(64 * c) * t.ld;
    const int64_t rows = t.rows - 64 * c;
    const float* b = t.bias;
    const int cols = t.cols;
    const int64_t ld = t.ld;
    const bool vec4 = ((reinterpret_cast<uintptr_t>(o) | (uintptr_t)(ld * 4)) & 15) == 0;
    store_staged<BN>(
        acc, stage, c, wq, lane,
        [&](int, int col, float v0, float v1) {
          if (b && col < cols) v0 += __ldg(b + col), v1 += __ldg(b + col + 1);
          return make_float2(v0, v1);
        },
        [&](int r, int col, float4 v) {
          if (r < rows && col < cols) {
            float* p = o + r * ld + col;
            if (vec4) {
              *reinterpret_cast<float4*>(p) = v;
            } else {
              *reinterpret_cast<float2*>(p) = make_float2(v.x, v.y);
              *reinterpret_cast<float2*>(p + 2) = make_float2(v.z, v.w);
            }
          }
        });
  }
};

template <int BN>
__global__ void __launch_bounds__(TILE_THREADS, 1) k_typed_linear_tc(const __grid_constant__ FwdJob job, int n_tiles) {
  split3_tile<BN, false, fwd_bk<BN>()>(job, n_tiles);
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

int make_map(CUtensorMap* m, const void* base, int64_t rows, int Kp, int box_rows, int kb) {
  EncodeTiledFn fn = get_encode_fn();
  HGT_REQUIRE(fn != nullptr, "hgt_typed_linear: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)Kp, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)Kp * 2};
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

// The tensor maps and the k-block count follow the kernel's k-block, fwd_bk<BN>().
template <int BN>
int launch_fwd(FwdJob& job, const __nv_bfloat16* const ops[4], int64_t a_rows, int64_t w_rows, int Kp, int tiles,
               cudaStream_t st) {
  constexpr int KB = fwd_bk<BN>();
  int rc;
  if ((rc = make_map(&job.a_hi, ops[0], a_rows, Kp, BM, KB))) return rc;
  if ((rc = make_map(&job.a_lo, ops[1], a_rows, Kp, BM, KB))) return rc;
  if ((rc = make_map(&job.w_hi, ops[2], w_rows, Kp, BN, KB))) return rc;
  if ((rc = make_map(&job.w_lo, ops[3], w_rows, Kp, BN, KB))) return rc;
  job.k_blocks = (Kp + KB - 1) / KB;
  const size_t smem = tile_smem_bytes<BN, KB>();
  HGT_CHECK_CUDA(cudaFuncSetAttribute(k_typed_linear_tc<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_typed_linear_tc<BN><<<persistent_grid(tiles), TILE_THREADS, smem, st>>>(job, tiles);
  HGT_LAUNCH_CHECK();
  return 0;
}

}  // namespace

bool hgt_typed_linear_tc_supported(int64_t lda, int32_t K, int32_t cb_width) {
  (void)lda;
  return cb_width % 16 == 0 && cb_width > 0 && K >= BK;
}

size_t hgt_typed_linear_tc_workspace(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K, int32_t cb_width) {
  int64_t a_rows, w_rows;
  extents(h_groups, n_groups, cb_width, &a_rows, &w_rows);
  const int Kp = (K + 7) / 8 * 8;
  return 4 * 256 + 2 * hgt_align_up((size_t)a_rows * Kp * 2, 256) + 2 * hgt_align_up((size_t)w_rows * Kp * 2, 256);
}

static int tc_run(const float* A, int64_t lda, const __nv_bfloat16* a_hi_in, const __nv_bfloat16* a_lo_in,
                  const float* W, const float* bias, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                  const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* cblocks, float* out,
                  void* workspace, size_t workspace_bytes, cudaStream_t st);

int hgt_typed_linear_tc(const float* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                        const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                        const hgt_lin_cblock* cblocks, float* out, void* workspace, size_t workspace_bytes,
                        cudaStream_t st) {
  return tc_run(A, lda, nullptr, nullptr, W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, workspace,
                workspace_bytes, st);
}

extern "C" int hgt_typed_linear_presplit_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K,
                                                         int32_t cb_width, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && (h_groups || n_groups == 0), "hgt_typed_linear_presplit_workspace_bytes: NULL argument");
  *out_bytes = n_groups > 0 ? hgt_typed_linear_tc_workspace(h_groups, n_groups, K, cb_width) : 0;
  return 0;
}

extern "C" int hgt_typed_linear_presplit(const void* a_hi, const void* a_lo, const float* W, const float* bias,
                                         int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                                         const hgt_lin_group* h_groups, int32_t n_groups,
                                         const hgt_lin_cblock* cblocks, float* out, void* workspace,
                                         size_t workspace_bytes, void* stream_) {
  HGT_REQUIRE(a_hi && a_lo, "hgt_typed_linear_presplit: NULL operand");
  HGT_REQUIRE(K % 8 == 0 && hgt_typed_linear_tc_supported(K, K, cb_width),
              "hgt_typed_linear_presplit: unsupported shape K=%d cb_width=%d", K, cb_width);
  if (n_groups == 0) return 0;
  if (n_groups > kMaxGroups) {                               // see hgt_typed_linear: chunked launches
    for (int g0 = 0; g0 < n_groups; g0 += kMaxGroups) {
      const int n = n_groups - g0 < kMaxGroups ? n_groups - g0 : kMaxGroups;
      int rc = hgt_typed_linear_presplit(a_hi, a_lo, W, bias, K, cb_width, groups + g0, h_groups + g0, n, cblocks, out,
                                         workspace, workspace_bytes, stream_);
      if (rc) return rc;
    }
    return 0;
  }
  return tc_run(nullptr, 0, reinterpret_cast<const __nv_bfloat16*>(a_hi), reinterpret_cast<const __nv_bfloat16*>(a_lo),
                W, bias, K, cb_width, groups, h_groups, n_groups, cblocks, out, workspace, workspace_bytes,
                (cudaStream_t)stream_);
}

static int tc_run(const float* A, int64_t lda, const __nv_bfloat16* a_hi_in, const __nv_bfloat16* a_lo_in,
                  const float* W, const float* bias, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                  const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* cblocks, float* out,
                  void* workspace, size_t workspace_bytes, cudaStream_t st) {
  HGT_REQUIRE(hgt_typed_linear_tc_supported(lda, K, cb_width), "hgt_typed_linear(tc): unsupported K=%d cb_width=%d", K,
              cb_width);
  const int Kp = (K + 7) / 8 * 8;
  int64_t a_rows, w_rows;
  extents(h_groups, n_groups, cb_width, &a_rows, &w_rows);
  size_t need = hgt_typed_linear_tc_workspace(h_groups, n_groups, K, cb_width);
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_typed_linear(tc): workspace too small (%zu < %zu)",
              workspace_bytes, need);
  char* p = reinterpret_cast<char*>(hgt_align_up(reinterpret_cast<size_t>(workspace), 256));
  __nv_bfloat16* a_hi = reinterpret_cast<__nv_bfloat16*>(p); p += hgt_align_up((size_t)a_rows * Kp * 2, 256);
  __nv_bfloat16* a_lo = reinterpret_cast<__nv_bfloat16*>(p); p += hgt_align_up((size_t)a_rows * Kp * 2, 256);
  __nv_bfloat16* w_hi = reinterpret_cast<__nv_bfloat16*>(p); p += hgt_align_up((size_t)w_rows * Kp * 2, 256);
  __nv_bfloat16* w_lo = reinterpret_cast<__nv_bfloat16*>(p);
  {
    int64_t n = a_rows * (Kp / 4);
    if (a_hi_in) {
      a_hi = const_cast<__nv_bfloat16*>(a_hi_in);            // split by the producer (e.g. the edge kernel)
      a_lo = const_cast<__nv_bfloat16*>(a_lo_in);
    } else if (n > 0) {
      k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(A, lda, a_rows, K, Kp, a_hi, a_lo);
      HGT_LAUNCH_CHECK();
    }
    n = w_rows * (Kp / 4);
    if (n > 0) k_split_bf16<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, K, w_rows, K, Kp, w_hi, w_lo);
    HGT_LAUNCH_CHECK();
  }
  FwdJob job;
  job.tile_n = pick_tile_n(cb_width);
  job.n_tiles_n = (cb_width + job.tile_n - 1) / job.tile_n;
  int64_t total = 0;
  for (int g = 0; g < n_groups; ++g) {
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
  job.n_groups = n_groups;
  job.cb_width = cb_width;
  const __nv_bfloat16* const ops[4] = {a_hi, a_lo, w_hi, w_lo};
  switch (job.tile_n) {
    case 64: return launch_fwd<64>(job, ops, a_rows, w_rows, Kp, (int)total, st);
    case 128: return launch_fwd<128>(job, ops, a_rows, w_rows, Kp, (int)total, st);
    default: return launch_fwd<256>(job, ops, a_rows, w_rows, Kp, (int)total, st);
  }
}
