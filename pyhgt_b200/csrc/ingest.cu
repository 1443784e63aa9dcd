// Device-side build of the sampler's adjacency blocks from typed edge arrays (pyhgt_b200/sampler.py:
// DeviceGraph.from_edges).  One block is fed by one edge array in insertion order: edge i gives target tgt[i] the
// neighbour src[i] at time time[i].  The block is the one FrozenGraph flattens from the dict `d[tgt[i]][src[i]] = time[i]`
// filled in array order (pyHGT/data.py:38-61, ogbn-mag/preprocess_ogbn_mag.py:29-42): rows in order of each target's
// first appearance, a row's neighbours in order of the pair's first appearance, a repeated pair keeping its first place
// and its last time.  All of it is stable radix sorts of edge positions (CUB) plus a few element-wise kernels:
//   sort pass: positions sorted by (target, source, position) -> group heads (one group per distinct pair) -> per group
//              its first and last position, per target its first position (the minimum over its groups);
//   write pass: targets sorted by first position -> row numbers and row_of; groups sorted by (row, first position) ->
//               ptr, nbr (the source of the first position) and time (the time of the last position).
#include "common.cuh"

#include <cub/block/block_reduce.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace {

constexpr int kThreads = 256;
constexpr int64_t kMaxEdges = (int64_t(1) << 31) - 1;     // positions are int32

struct IngestScratch {
  uint64_t *a8, *b8, *c8;                       // sort keys (two buffers) and the group-head scan
  int32_t *p4, *q4;                             // sorted positions (two buffers)
  int32_t *gfirst, *glast, *gtord, *tfirst;     // per group: first / last position, target ordinal; per target: first
  void* cub_tmp;
  size_t cub_bytes;
};

size_t carve(IngestScratch& s, void* base, int64_t n) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += hgt_align_up(bytes, 256);
    return base ? (char*)base + o : (char*)nullptr;
  };
  const size_t m = (size_t)(n > 0 ? n : 1);
  s.a8 = (uint64_t*)take(8 * m);
  s.b8 = (uint64_t*)take(8 * m);
  s.c8 = (uint64_t*)take(8 * m);
  s.p4 = (int32_t*)take(4 * m);
  s.q4 = (int32_t*)take(4 * m);
  s.gfirst = (int32_t*)take(4 * m);
  s.glast = (int32_t*)take(4 * m);
  s.gtord = (int32_t*)take(4 * m);
  s.tfirst = (int32_t*)take(4 * m);
  size_t b1 = 0, b2 = 0, b3 = 0;
  cub::DoubleBuffer<uint64_t> k8(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> k4(nullptr, nullptr);
  cub::DoubleBuffer<int32_t> v4(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, b1, k8, v4, (int)m);
  cub::DeviceRadixSort::SortPairs(nullptr, b2, k4, v4, (int)m);
  cub::DeviceScan::InclusiveSum(nullptr, b3, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)m);
  s.cub_bytes = b1 > b2 ? b1 : b2;
  s.cub_bytes = s.cub_bytes > b3 ? s.cub_bytes : b3;
  s.cub_tmp = take(s.cub_bytes);
  return off;
}

// bits that hold every value in [0, v]
int bits_for(int64_t v) {
  int b = 1;
  while (b < 63 && (int64_t(1) << b) <= v) ++b;
  return b;
}

inline unsigned grid_for(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads > 0 ? (n + kThreads - 1) / kThreads : 1); }

__global__ void k_init(const int64_t* __restrict__ src, int64_t n, uint64_t* __restrict__ key, int32_t* __restrict__ pos,
                       int32_t* __restrict__ tfirst, int64_t* __restrict__ stats) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    stats[0] = stats[1] = 0;
    stats[2] = INT64_MAX;
    stats[3] = INT64_MIN;
  }
  if (i >= n) return;
  key[i] = (uint64_t)src[i];
  pos[i] = (int32_t)i;
  tfirst[i] = INT32_MAX;
}

__global__ void k_gather_targets(const int64_t* __restrict__ tgt, const int32_t* __restrict__ pos, int64_t n,
                                 uint64_t* __restrict__ key) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) key[i] = (uint64_t)tgt[pos[i]];
}

// heads[i] = (target head << 32) | group head, in (target, source, position) order; its inclusive scan numbers both.
__global__ void k_heads(const uint64_t* __restrict__ tkey, const int64_t* __restrict__ src,
                        const int32_t* __restrict__ pos, int64_t n, uint64_t* __restrict__ heads) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool th = i == 0 || tkey[i] != tkey[i - 1];
  const bool gh = th || src[pos[i]] != src[pos[i - 1]];
  heads[i] = ((uint64_t)th << 32) | (uint64_t)gh;
}

__global__ void k_groups(const uint64_t* __restrict__ scan, const int32_t* __restrict__ pos,
                         const int64_t* __restrict__ time, int64_t n, int32_t* __restrict__ gfirst,
                         int32_t* __restrict__ glast, int32_t* __restrict__ gtord, int32_t* __restrict__ tfirst,
                         int64_t* __restrict__ stats) {
  using Reduce = cub::BlockReduce<long long, kThreads>;
  __shared__ typename Reduce::TempStorage red;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  long long lo = INT64_MAX, hi = INT64_MIN;
  if (i < n) {
    const uint64_t s = scan[i];
    const uint64_t d = s - (i ? scan[i - 1] : 0ull);
    const int32_t g = (int32_t)(uint32_t)s - 1, t = (int32_t)(s >> 32) - 1, p = pos[i];
    if ((uint32_t)d) {
      gfirst[g] = p;
      gtord[g] = t;
      atomicMin(tfirst + t, p);
    }
    if (i == n - 1 || (uint32_t)(scan[i + 1] - s)) {       // last of its group: the time the dict keeps
      glast[g] = p;
      if (time) lo = hi = time[p];
    }
    if (i == n - 1) {
      stats[0] = t + 1;
      stats[1] = g + 1;
    }
  }
  if (!time) return;
  const long long blo = Reduce(red).Reduce(lo, cub::Min());
  __syncthreads();
  const long long bhi = Reduce(red).Reduce(hi, cub::Max());
  if (threadIdx.x == 0 && blo <= bhi) {
    atomicMin((long long*)stats + 2, blo);
    atomicMax((long long*)stats + 3, bhi);
  }
}

__global__ void k_iota(int32_t* __restrict__ v, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = (int32_t)i;
}

template <typename T>
__global__ void k_fill(T* __restrict__ a, int64_t n, T v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// row r is the target whose first position is the r-th smallest
template <typename T>
__global__ void k_rows(const uint32_t* __restrict__ first_sorted, const int32_t* __restrict__ order,
                       const int64_t* __restrict__ tgt, int64_t n_rows, int32_t* __restrict__ rank,
                       T* __restrict__ row_of) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  rank[order[r]] = (int32_t)r;
  row_of[tgt[first_sorted[r]]] = (T)r;
}

__global__ void k_group_keys(const int32_t* __restrict__ gtord, const int32_t* __restrict__ gfirst,
                             const int32_t* __restrict__ rank, int64_t n_groups, uint64_t* __restrict__ key,
                             int32_t* __restrict__ val) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  key[g] = ((uint64_t)(uint32_t)rank[gtord[g]] << 32) | (uint32_t)gfirst[g];
  val[g] = (int32_t)g;
}

// entry i of the CSR: the i-th group in (row, first position) order; every row has at least one entry
template <typename T>
__global__ void k_write(const uint64_t* __restrict__ key, const int32_t* __restrict__ val,
                        const int32_t* __restrict__ gfirst, const int32_t* __restrict__ glast,
                        const int64_t* __restrict__ src, const int64_t* __restrict__ time, int64_t n_groups,
                        int64_t n_rows, T no_time, T* __restrict__ ptr, T* __restrict__ nbr, T* __restrict__ tout) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_groups) return;
  const int32_t g = val[i];
  nbr[i] = (T)src[gfirst[g]];
  tout[i] = time ? (T)time[glast[g]] : no_time;
  const uint64_t row = key[i] >> 32;
  if (i == 0 || (key[i - 1] >> 32) != row) ptr[row] = (T)i;
  if (i == n_groups - 1) ptr[n_rows] = (T)n_groups;
}

template <typename T>
int write_block(const IngestScratch& s, const int64_t* tgt, const int64_t* src, const int64_t* time, int64_t n,
                int64_t n_rows, int64_t n_groups, T no_time, T* row_of, int64_t n_row_of, T* ptr, T* nbr, T* tout,
                cudaStream_t st) {
  if (n_row_of > 0) {
    k_fill<T><<<grid_for(n_row_of), kThreads, 0, st>>>(row_of, n_row_of, (T)-1);
    HGT_LAUNCH_CHECK();
  }
  if (n == 0) {
    HGT_CHECK_CUDA(cudaMemsetAsync(ptr, 0, sizeof(T), st));
    return 0;
  }
  size_t tmp = s.cub_bytes;
  // rows: targets by first position
  k_iota<<<grid_for(n_rows), kThreads, 0, st>>>(s.p4, n_rows);
  HGT_LAUNCH_CHECK();
  cub::DoubleBuffer<uint32_t> fk((uint32_t*)s.tfirst, (uint32_t*)s.a8);
  cub::DoubleBuffer<int32_t> ov(s.p4, s.q4);
  HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, fk, ov, (int)n_rows, 0, bits_for(n - 1), st));
  int32_t* rank = (int32_t*)s.b8;
  k_rows<T><<<grid_for(n_rows), kThreads, 0, st>>>(fk.Current(), ov.Current(), tgt, n_rows, rank, row_of);
  HGT_LAUNCH_CHECK();
  // entries: groups by (row, first position)
  k_group_keys<<<grid_for(n_groups), kThreads, 0, st>>>(s.gtord, s.gfirst, rank, n_groups, s.c8, s.p4);
  HGT_LAUNCH_CHECK();
  cub::DoubleBuffer<uint64_t> gk(s.c8, s.a8);
  cub::DoubleBuffer<int32_t> gv(s.p4, s.q4);
  tmp = s.cub_bytes;
  HGT_CHECK_CUDA(
      cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, gk, gv, (int)n_groups, 0, 32 + bits_for(n_rows - 1), st));
  k_write<T><<<grid_for(n_groups), kThreads, 0, st>>>(gk.Current(), gv.Current(), s.gfirst, s.glast, src, time, n_groups,
                                                      n_rows, no_time, ptr, nbr, tout);
  HGT_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int hgt_ingest_workspace_bytes(int64_t n_edges, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_edges >= 0 && n_edges <= kMaxEdges,
              "hgt_ingest_workspace_bytes: n_edges must lie in [0, 2^31 - 1], got %lld", (long long)n_edges);
  IngestScratch s;
  *out_bytes = carve(s, nullptr, n_edges);
  return 0;
}

extern "C" int hgt_ingest_block_sort(const int64_t* tgt, const int64_t* src, const int64_t* time, int64_t n_edges,
                                     int64_t tgt_max, int64_t src_max, int64_t* stats, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(n_edges >= 0 && n_edges <= kMaxEdges && stats && workspace && (n_edges == 0 || (tgt && src)) &&
                  tgt_max >= 0 && src_max >= 0,
              "hgt_ingest_block_sort: bad arguments");
  IngestScratch s;
  const size_t need = carve(s, nullptr, n_edges);
  HGT_REQUIRE(workspace_bytes >= need, "hgt_ingest_block_sort: workspace of %zu bytes, %zu needed", workspace_bytes,
              need);
  carve(s, workspace, n_edges);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = n_edges;
  k_init<<<grid_for(n), kThreads, 0, st>>>(src, n, s.a8, s.p4, s.tfirst, stats);
  HGT_LAUNCH_CHECK();
  if (n == 0) return 0;
  // (target, source, position): a stable sort by source, then a stable sort by target
  cub::DoubleBuffer<uint64_t> keys(s.a8, s.b8);
  cub::DoubleBuffer<int32_t> pos(s.p4, s.q4);
  size_t tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, keys, pos, (int)n, 0, bits_for(src_max), st));
  k_gather_targets<<<grid_for(n), kThreads, 0, st>>>(tgt, pos.Current(), n, keys.Current());
  HGT_LAUNCH_CHECK();
  tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, keys, pos, (int)n, 0, bits_for(tgt_max), st));
  k_heads<<<grid_for(n), kThreads, 0, st>>>(keys.Current(), src, pos.Current(), n, s.c8);
  HGT_LAUNCH_CHECK();
  tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceScan::InclusiveSum(s.cub_tmp, tmp, s.c8, keys.Alternate(), (int)n, st));
  k_groups<<<grid_for(n), kThreads, 0, st>>>(keys.Alternate(), pos.Current(), time, n, s.gfirst, s.glast, s.gtord,
                                             s.tfirst, stats);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_ingest_block_write(const int64_t* tgt, const int64_t* src, const int64_t* time, int64_t n_edges,
                                      int64_t n_rows, int64_t n_entries, int32_t narrow, int64_t no_time, void* row_of,
                                      int64_t n_row_of, void* ptr, void* nbr, void* time_out, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(n_edges >= 0 && n_edges <= kMaxEdges && n_rows >= 0 && n_entries >= n_rows && n_entries <= n_edges &&
                  (n_edges == 0) == (n_rows == 0) && n_row_of >= 0 && (n_row_of == 0 || row_of) && ptr && workspace &&
                  (n_edges == 0 || (tgt && src && nbr && time_out)),
              "hgt_ingest_block_write: bad arguments");
  IngestScratch s;
  const size_t need = carve(s, nullptr, n_edges);
  HGT_REQUIRE(workspace_bytes >= need, "hgt_ingest_block_write: workspace of %zu bytes, %zu needed", workspace_bytes,
              need);
  carve(s, workspace, n_edges);
  cudaStream_t st = (cudaStream_t)stream;
  if (narrow)
    return write_block<int32_t>(s, tgt, src, time, n_edges, n_rows, n_entries, INT32_MIN, (int32_t*)row_of, n_row_of,
                                (int32_t*)ptr, (int32_t*)nbr, (int32_t*)time_out, st);
  return write_block<int64_t>(s, tgt, src, time, n_edges, n_rows, n_entries, no_time, (int64_t*)row_of, n_row_of,
                              (int64_t*)ptr, (int64_t*)nbr, (int64_t*)time_out, st);
}
