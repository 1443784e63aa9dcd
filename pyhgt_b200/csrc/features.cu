// Node features derived from the sampler's adjacency blocks (pyhgt_b200/sampler.py: mag_features), the ogbn-mag
// preprocessing rules of preprocess_ogbn_mag.py:45-99 over the dict graph the blocks are a CSR form of:
//   degree pass:          deg[id] = sum over the given blocks of id's row length; out[id * ld] = log10(deg[id]);
//   neighbour-mean pass:  out[id] = (sum over the given blocks, in order, of the source rows of id's row) / pair count,
//                         zero for an id with no pairs.
// A block is read at its own width (HGT_BLOCK_NARROW) and wherever its arrays live: a host-placed block's addresses are
// mapped host memory, read in place as the sampler kernels read them.  Every sum runs in one fixed order (integers for
// the degree, one lane per column in block and row order for the means), so both passes are bitwise repeatable.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kUnroll = 4;          // source rows a lane has in flight

__device__ __forceinline__ bool narrow_of(const hgt_gsample_block& b) { return b.skip & HGT_BLOCK_NARROW; }
__device__ __forceinline__ int64_t idx_at(const int64_t* a, bool narrow, int64_t i) {
  return narrow ? (int64_t)reinterpret_cast<const int32_t*>(a)[i] : a[i];
}

// [begin, end) of id's row in block b; begin == end when the block has no row for id.
__device__ __forceinline__ void row_span(const hgt_gsample_block& b, int64_t id, int64_t& begin, int64_t& end) {
  begin = end = 0;
  if (id >= b.n_row_of) return;
  const bool nw = narrow_of(b);
  const int64_t r = idx_at(b.row_of, nw, id);
  if (r < 0) return;
  begin = idx_at(b.ptr, nw, r);
  end = idx_at(b.ptr, nw, r + 1);
}

__global__ void __launch_bounds__(kThreads) k_degree(const hgt_gsample_block* __restrict__ blocks, int32_t n_blocks,
                                                     int64_t n_nodes, int64_t* __restrict__ deg, float* __restrict__ out,
                                                     int64_t ld) {
  const int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n_nodes) return;
  int64_t d = 0;
  for (int32_t b = 0; b < n_blocks; ++b) {
    int64_t begin, end;
    row_span(blocks[b], id, begin, end);
    d += end - begin;
  }
  deg[id] = d;
  out[id * ld] = (float)log10((double)d);            // log10(0) = -inf, as numpy gives
}

// V consecutive source columns as doubles.
template <int V>
__device__ __forceinline__ void load_cols(const float* p, double (&v)[V]) {
  if constexpr (V == 4) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j) v[j] = p[j];
  }
}
template <int V>
__device__ __forceinline__ void load_cols(const double* p, double (&v)[V]) {
  if constexpr (V == 4) {
    const double2 a = reinterpret_cast<const double2*>(p)[0], b = reinterpret_cast<const double2*>(p)[1];
    v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
  } else {
#pragma unroll
    for (int j = 0; j < V; ++j) v[j] = p[j];
  }
}

// One warp per target id.  Lane l owns columns [c + V l, c + V l + V) of each 32 V-column tile c; the warp walks the
// id's rows block by block, 32 neighbour ids per coalesced read, kUnroll source rows in flight per lane, and adds them
// into the lane's fp64 sums in block and row order.  V = 4 needs feat_dim and src_ld to be multiples of 4 and src
// 16-byte aligned (one vector load per lane and row); V = 1 takes any layout.
template <typename S, int V>
__global__ void __launch_bounds__(kThreads) k_neighbour_mean(const hgt_gsample_block* __restrict__ blocks,
                                                             int32_t n_blocks, int64_t n_nodes, const S* __restrict__ src,
                                                             int64_t src_ld, int32_t feat_dim, double* __restrict__ out64,
                                                             int64_t ld64, float* __restrict__ out32, int64_t ld32) {
  const int lane = threadIdx.x & 31;
  const int64_t id = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (id >= n_nodes) return;
  for (int c = 0; c < feat_dim; c += 32 * V) {
    const int col = c + V * lane;
    const bool mine = col < feat_dim;                  // V = 4: feat_dim % 4 == 0, so a lane's columns are all in
    const int lcol = mine ? col : 0;                   // a lane past the last column reads column 0 and writes nothing
    double acc[V];
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] = 0.0;
    int64_t pairs = 0;
    for (int32_t b = 0; b < n_blocks; ++b) {
      const hgt_gsample_block blk = blocks[b];
      int64_t begin, end;
      row_span(blk, id, begin, end);
      pairs += end - begin;
      const bool nw = narrow_of(blk);
      for (int64_t e0 = begin; e0 < end; e0 += 32) {
        const int n = end - e0 < 32 ? (int)(end - e0) : 32;
        const int64_t my_nbr = lane < n ? idx_at(blk.nbr, nw, e0 + lane) : 0;
        int k = 0;
        for (; k + kUnroll <= n; k += kUnroll) {
          double v[kUnroll][V];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const int64_t s = __shfl_sync(0xffffffffu, my_nbr, k + u);
            load_cols<V>(src + s * src_ld + lcol, v[u]);
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u)
#pragma unroll
            for (int j = 0; j < V; ++j) acc[j] += v[u][j];
        }
        for (; k < n; ++k) {
          const int64_t s = __shfl_sync(0xffffffffu, my_nbr, k);
          double v[V];
          load_cols<V>(src + s * src_ld + lcol, v);
#pragma unroll
          for (int j = 0; j < V; ++j) acc[j] += v[j];
        }
      }
    }
    if (!mine) continue;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const double m = pairs ? acc[j] / (double)pairs : 0.0;
      if (out64) out64[id * ld64 + col + j] = m;
      if (out32) out32[id * ld32 + col + j] = (float)m;
    }
  }
}

template <typename S>
int launch_mean(const hgt_gsample_block* blocks, int32_t n_blocks, int64_t n_nodes, const S* src, int64_t src_ld,
                int32_t feat_dim, double* out64, int64_t ld64, float* out32, int64_t ld32, cudaStream_t st) {
  const unsigned grid = (unsigned)((n_nodes + kWarps - 1) / kWarps);
  const bool vec = feat_dim % 4 == 0 && src_ld % 4 == 0 && (uintptr_t)src % 16 == 0;
  if (vec)
    k_neighbour_mean<S, 4><<<grid, kThreads, 0, st>>>(blocks, n_blocks, n_nodes, src, src_ld, feat_dim, out64, ld64,
                                                      out32, ld32);
  else
    k_neighbour_mean<S, 1><<<grid, kThreads, 0, st>>>(blocks, n_blocks, n_nodes, src, src_ld, feat_dim, out64, ld64,
                                                      out32, ld32);
  HGT_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int hgt_feat_degree(const hgt_gsample_block* blocks, int32_t n_blocks, int64_t n_nodes, int64_t* deg,
                               float* out, int64_t ld_out, void* stream) {
  HGT_REQUIRE(n_blocks >= 0 && (n_blocks == 0 || blocks) && n_nodes >= 0 && ld_out >= 1 &&
                  (n_nodes == 0 || (deg && out)) && (n_nodes + 255) / 256 <= INT32_MAX,
              "hgt_feat_degree: bad arguments (n_blocks %d, n_nodes %lld, ld_out %lld)", n_blocks,
              (long long)n_nodes, (long long)ld_out);
  if (n_nodes == 0) return 0;
  k_degree<<<(unsigned)((n_nodes + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      blocks, n_blocks, n_nodes, deg, out, ld_out);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_feat_neighbour_mean(const hgt_gsample_block* blocks, int32_t n_blocks, int64_t n_nodes,
                                       const void* src, int32_t src_fp64, int64_t src_ld, int32_t feat_dim,
                                       double* out64, int64_t ld64, float* out32, int64_t ld32, void* stream) {
  HGT_REQUIRE(n_blocks >= 0 && (n_blocks == 0 || blocks) && n_nodes >= 0 && feat_dim >= 1 && src_ld >= feat_dim &&
                  (out64 || out32) && (!out64 || ld64 >= feat_dim) && (!out32 || ld32 >= feat_dim) &&
                  (n_nodes == 0 || n_blocks == 0 || src) && (n_nodes + kWarps - 1) / kWarps <= INT32_MAX,
              "hgt_feat_neighbour_mean: bad arguments (n_blocks %d, n_nodes %lld, feat_dim %d, src_ld %lld, "
              "ld64 %lld, ld32 %lld)", n_blocks, (long long)n_nodes, feat_dim, (long long)src_ld, (long long)ld64,
              (long long)ld32);
  if (n_nodes == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (src_fp64)
    return launch_mean<double>(blocks, n_blocks, n_nodes, (const double*)src, src_ld, feat_dim, out64, ld64, out32,
                               ld32, st);
  return launch_mean<float>(blocks, n_blocks, n_nodes, (const float*)src, src_ld, feat_dim, out64, ld64, out32, ld32,
                            st);
}
