// Disjoint union of B sampled batches in the to_torch layout (pyhgt_b200/sampler.py: merge_batches).  The union is
// type-major: type 0 rows of member 0, of member 1, ..., then type 1 rows, ... so node_type stays sorted and the
// sync-free plan applies.  Member b's type-t rows [loc_off, loc_off + count) map to union rows uoff[b, t] + (i - loc_off);
// edges keep their member order, member after member.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

inline int64_t blocks_for(int64_t n, int per = kThreads) { return (n + per - 1) / per; }

// Union row of member-local row v (-1 when v is not a row of the member: the union plan's range check reports it).
__device__ __forceinline__ int64_t union_row(const int64_t* loc_off, const int64_t* uoff, int T, int64_t v) {
  if (v < 0 || v >= loc_off[T]) return -1;
  int t = 0;
  while (t + 1 < T && v >= loc_off[t + 1]) ++t;
  return uoff[t] + v - loc_off[t];
}

// One warp per <member (grid.y), local row i>: node_type, the member's row map and the feature row (FeatT: float, or
// uint16_t for bf16 rows, copied as they are).
template <class FeatT>
__global__ void k_merge_nodes(const hgt_merge_member* members, int32_t T, const int64_t* loc_off, const int64_t* uoff,
                              int32_t feat_dim, int64_t* node_type, FeatT* node_feature, int64_t* member_rows) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const hgt_merge_member mb = members[b];
  const int64_t* lo = loc_off + (int64_t)b * (T + 1);
  if (i >= lo[T]) return;
  int t = 0;
  while (t + 1 < T && i >= lo[t + 1]) ++t;
  const int64_t u = uoff[(int64_t)b * T + t] + i - lo[t];
  if (lane == 0) {
    node_type[u] = t;
    member_rows[mb.node_base + i] = u;
  }
  if (node_feature) {
    const FeatT* src = reinterpret_cast<const FeatT*>(mb.node_feature) + i * (int64_t)feat_dim;
    FeatT* dst = node_feature + u * (int64_t)feat_dim;
    for (int c = lane; c < feat_dim; c += 32) dst[c] = src[c];
  }
}

// One thread per <member (grid.y), edge e>: endpoints remapped by (member, type) offset, type and time copied.
__global__ void k_merge_edges(const hgt_merge_member* members, int32_t T, const int64_t* loc_off, const int64_t* uoff,
                              int64_t n_edges, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  const hgt_merge_member mb = members[b];
  if (e >= mb.n_edges) return;
  const int64_t* lo = loc_off + (int64_t)b * (T + 1);
  const int64_t* uo = uoff + (int64_t)b * T;
  const int64_t o = mb.edge_base + e;
  edge_index[o] = union_row(lo, uo, T, mb.edge_index[e]);
  edge_index[n_edges + o] = union_row(lo, uo, T, mb.edge_index[mb.n_edges + e]);
  edge_type[o] = mb.edge_type[e];
  edge_time[o] = mb.edge_time[e];
}

template <class FeatT>
int merge_batches(const hgt_merge_member* members, int32_t n_members, int32_t num_types, const int64_t* loc_off,
                  const int64_t* uoff, int64_t max_rows, int64_t max_edges, int64_t n_edges, int32_t feat_dim,
                  int64_t* node_type, FeatT* node_feature, int64_t* member_rows, int64_t* edge_index,
                  int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(members && n_members >= 0 && n_members < 65536 && num_types > 0 && max_rows >= 0 && max_edges >= 0 &&
                  n_edges >= 0 && feat_dim >= 0,
              "hgt_merge_batches: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (n_members == 0) return 0;
  if (max_rows > 0) {
    k_merge_nodes<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_members), kThreads, 0, st>>>(
        members, num_types, loc_off, uoff, feat_dim, node_type, node_feature, member_rows);
    HGT_LAUNCH_CHECK();
  }
  if (max_edges > 0) {
    k_merge_edges<<<dim3((unsigned)blocks_for(max_edges), n_members), kThreads, 0, st>>>(
        members, num_types, loc_off, uoff, n_edges, edge_index, edge_type, edge_time);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace

extern "C" int hgt_merge_batches(const hgt_merge_member* members, int32_t n_members, int32_t num_types,
                                 const int64_t* loc_off, const int64_t* uoff, int64_t max_rows, int64_t max_edges,
                                 int64_t n_edges, int32_t feat_dim, int64_t* node_type, float* node_feature,
                                 int64_t* member_rows, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time,
                                 void* stream) {
  return merge_batches(members, n_members, num_types, loc_off, uoff, max_rows, max_edges, n_edges, feat_dim, node_type,
                       node_feature, member_rows, edge_index, edge_type, edge_time, stream);
}

extern "C" int hgt_merge_batches_bf16(const hgt_merge_member* members, int32_t n_members, int32_t num_types,
                                      const int64_t* loc_off, const int64_t* uoff, int64_t max_rows, int64_t max_edges,
                                      int64_t n_edges, int32_t feat_dim, int64_t* node_type, void* node_feature,
                                      int64_t* member_rows, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time,
                                      void* stream) {
  return merge_batches(members, n_members, num_types, loc_off, uoff, max_rows, max_edges, n_edges, feat_dim, node_type,
                       static_cast<uint16_t*>(node_feature), member_rows, edge_index, edge_type, edge_time, stream);
}
