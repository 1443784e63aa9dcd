// HGSampling on the GPU (reference pyHGT/data.py:87-256: sample_subgraph + to_torch), the device path of
// pyhgt_b200/sampler.py:sample_subgraph_cuda.  Draws from the same distribution as the host sampler (which replays numpy's
// stream bit for bit) with a counter-based RNG (Philox), so the result is a function of (seed, inputs) alone:
//   * add_budget (data.py:108-130) for a whole batch of targets: one warp per <target, block> segment draws the ordered
//     uniform subset (Floyd's set + Fisher-Yates order == permutation(n)[:k]) and applies the filters; the budget is
//     updated with order-independent atomics (fixed-point score, max / min of the candidate's position in the
//     reference's processing order for the last-writer time and the first-entry stamp), so it is bitwise repeatable;
//   * selection (data.py:150-165): Efraimidis-Spirakis keys log(u)/score^2 sorted with CUB (same ordered distribution as
//     np.random.choice(p, replace=False)), or the insertion stamp when the budget is smaller than the width;
//   * rebuild (data.py:181-209) + to_torch layout (data.py:226-256): count / scan / write per adjacency block.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <curand_kernel.h>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr double kScoreScale = 1099511627776.0;          // 2^40: budget scores are fixed point (deterministic sums)
constexpr long long kNoSeq = 0x7fffffffffffffffLL;
constexpr unsigned kFull = 0xffffffffu;
constexpr uint64_t kSelectStream = 0x5e1ec7ULL << 40;     // keeps selection draws apart from neighbour draws

__device__ __forceinline__ uint64_t rnd64(curandStatePhilox4_32_10_t* s) {
  const uint64_t hi = curand(s);
  return (hi << 32) | curand(s);
}
// uniform in [0, m): multiply-high of a 64-bit draw (bias below m / 2^64)
__device__ __forceinline__ int64_t rnd_below(curandStatePhilox4_32_10_t* s, int64_t m) {
  return (int64_t)__umul64hi(rnd64(s), (uint64_t)m);
}

__device__ __forceinline__ int64_t seg_size(const hgt_gsample_block& blk, int64_t tid, int64_t width, int64_t* a,
                                            int64_t* deg) {
  *a = 0;
  *deg = 0;
  if (blk.skip || tid < 0 || tid >= blk.n_row_of) return 0;             // 'self' (data.py:116), or no adjacency
  const int64_t row = blk.row_of[tid];
  if (row < 0) return 0;
  *a = blk.ptr[row];
  *deg = blk.ptr[row + 1] - *a;
  return *deg < width ? *deg : width;                                   // data.py:119-122
}

__global__ void k_seg_count(const hgt_gsample_block* blocks, int32_t n_blocks, const int64_t* tgt_id, int64_t max_targets,
                            const int64_t* n_targets, int64_t width, int64_t* seg_cnt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t n_seg = max_targets * n_blocks;
  if (i > n_seg) return;
  if (i == n_seg) { seg_cnt[i] = 0; return; }
  const int64_t k = i / n_blocks;
  const int64_t n = n_targets ? *n_targets : max_targets;
  int64_t a, deg;
  seg_cnt[i] = k < n ? seg_size(blocks[i % n_blocks], tgt_id[k], width, &a, &deg) : 0;
}

// One warp per <target k, block b>.  seq = seg_off + j is the candidate's position in the reference's processing order
// (target, block, neighbour in subset order), the key of every order-dependent rule.
__global__ void k_candidates(hgt_gsample_state st, const hgt_gsample_block* blocks, int32_t n_blocks,
                             const int64_t* tgt_id, const int64_t* tgt_time, int64_t max_targets,
                             const int64_t* seg_cnt, const int64_t* seg_off, int64_t width, int32_t time_filter,
                             int64_t max_time, int64_t no_time, uint64_t seed, int64_t step, int64_t* cand_pos,
                             int64_t* cand_slot, int64_t* cand_time, int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (seg >= max_targets * n_blocks) return;
  const int64_t n_s = seg_cnt[seg];
  if (n_s == 0) return;
  const int64_t k = seg / n_blocks;
  const hgt_gsample_block blk = blocks[seg % n_blocks];
  int64_t a, deg;
  seg_size(blk, tgt_id[k], width, &a, &deg);
  const int64_t off = seg_off[seg];
  int64_t* S = cand_pos + off;
  const bool all = deg < width;
  if (!all) {
    // Floyd: a uniform n_s-subset of [0, deg); then a uniform order (Fisher-Yates).  Every lane runs the same stream.
    curandStatePhilox4_32_10_t rs;
    curand_init(seed, ((uint64_t)step << 32) | (uint64_t)seg, 0, &rs);
    for (int64_t c = 0, jj = deg - n_s; jj < deg; ++jj, ++c) {
      const int64_t t = rnd_below(&rs, jj + 1);
      bool found = false;
      for (int64_t q = lane; q < c; q += 32) found |= (S[q] == t);
      found = __any_sync(kFull, found);
      if (lane == 0) S[c] = found ? jj : t;
      __syncwarp();
    }
    if (lane == 0)
      for (int64_t i = n_s - 1; i > 0; --i) {
        const int64_t j = rnd_below(&rs, i + 1);
        const int64_t x = S[i];
        S[i] = S[j];
        S[j] = x;
      }
    __syncwarp();
  }
  const int64_t target_time = tgt_time[k];
  const int src = blk.src_type;
  const int64_t base = st.type_off[src], n_ids = st.type_off[src + 1] - base;
  const unsigned long long w = (unsigned long long)llrint(kScoreScale / (double)n_s);   // 1. / len(sampled_ids)
  for (int64_t j = lane; j < n_s; j += 32) {
    const int64_t seq = off + j;
    const int64_t pos = a + (all ? j : S[j]);
    const int64_t sid = blk.nbr[pos];
    int64_t tm = blk.time[pos];
    if (tm == no_time) tm = target_time;                                // data.py:125-126
    cand_slot[seq] = -1;
    if (time_filter && tm > max_time) continue;                         // data.py:127, first operand of the `or`
    atomicMin((long long*)&st.type_min[2 * src], (long long)seq);      // layer_data[source_type] springs into being
    if (sid < 0 || sid >= n_ids) { flags[0] = 1; continue; }
    const int64_t slot = base + sid;
    if (st.ser[slot] >= 0) continue;                                    // already sampled
    atomicMin((long long*)&st.type_min[2 * src + 1], (long long)seq);  // budget[source_type] springs into being
    atomicAdd(&st.score[slot], w);
    atomicMax((long long*)&st.last_seq[slot], (long long)seq);
    if (st.bstamp[slot] < 0) atomicMin((long long*)&st.first_seq[slot], (long long)seq);
    cand_slot[seq] = slot;
    cand_time[seq] = tm;
  }
}

// The candidate that wrote last sets the budget time (data.py:130); the first one of a new entry sets its stamp.  The
// matching candidate also resets the scratch word: no other candidate of the slot can match either value.
__global__ void k_resolve(hgt_gsample_state st, const int64_t* seg_off, int64_t n_seg, int64_t cap,
                          const int64_t* cand_slot, const int64_t* cand_time, int64_t stamp_base) {
  const int64_t seq = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (seq >= cap || seq >= seg_off[n_seg]) return;
  const int64_t slot = cand_slot[seq];
  if (slot < 0) return;
  if (st.last_seq[slot] == seq) {
    st.btime[slot] = cand_time[seq];
    st.last_seq[slot] = -1;
  }
  if (st.first_seq[slot] == seq) {
    st.bstamp[slot] = stamp_base + seq;
    st.first_seq[slot] = kNoSeq;
  }
}

// First-touch numbers of layer_data[t] / budget[t] (the key orders of the reference's defaultdicts): types touched for
// the first time in this step are numbered in the order of their first qualifying candidate.
__global__ void k_touch(hgt_gsample_state st) {
  for (int kind = 0; kind < 2; ++kind) {
    for (;;) {
      int best = -1;
      long long bv = kNoSeq;
      for (int t = 0; t < st.num_types; ++t)
        if (st.type_seq[2 * t + kind] < 0 && st.type_min[2 * t + kind] < bv) { bv = st.type_min[2 * t + kind]; best = t; }
      if (best < 0) break;
      st.type_seq[2 * best + kind] = st.counters[kind]++;
    }
    for (int t = 0; t < st.num_types; ++t) st.type_min[2 * t + kind] = kNoSeq;
  }
}

__global__ void k_sel_count(hgt_gsample_state st, int32_t type, unsigned long long* count) {
  const int64_t base = st.type_off[type], n = st.type_off[type + 1] - base;
  unsigned long long c = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    c += st.bstamp[base + i] >= 0;
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

// Sort keys (descending): budget smaller than the width -> every entry in insertion order (key -stamp); otherwise
// Efraimidis-Spirakis log(u) / score^2 (data.py:158-160).  Entries outside the budget sort last.
__global__ void k_sel_keys(hgt_gsample_state st, int32_t type, int64_t width, const unsigned long long* count,
                           uint64_t seed, int64_t step, double* keys, int32_t* vals) {
  const int64_t base = st.type_off[type], n = st.type_off[type + 1] - base;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t slot = base + i;
  const int64_t stamp = st.bstamp[slot];
  double key = -INFINITY;
  if (stamp >= 0) {
    if (width > (int64_t)*count) {
      key = -(double)stamp;
    } else {
      curandStatePhilox4_32_10_t rs;
      curand_init(seed ^ kSelectStream, ((uint64_t)step << 40) | (uint64_t)i, 0, &rs);
      const double u = (double)((rnd64(&rs) >> 11) + 1) * 0x1.0p-53;   // (0, 1]
      const double s = (double)st.score[slot] / kScoreScale;
      key = log(u) / (s * s);
    }
  }
  keys[i] = key;
  vals[i] = (int32_t)i;
}

// data.py:166-170: the chosen ids join layer_data in key order (ser), become the next add_budget's targets, and leave
// the budget.
__global__ void k_sel_take(hgt_gsample_state st, int32_t type, int64_t width, const unsigned long long* count,
                           const int32_t* vals, int64_t* tgt_id, int64_t* tgt_time, int32_t* flags) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t m = (int64_t)*count < width ? (int64_t)*count : width;
  if (r >= m) return;
  const int64_t i = vals[r];
  const int64_t slot = st.type_off[type] + i;
  const int64_t ser = st.n_layer[type] + r;
  if (st.lid_off[type] + ser >= st.lid_off[type + 1]) { flags[0] = 1; return; }
  st.ser[slot] = (int32_t)ser;
  st.ltime[slot] = st.btime[slot];
  st.lid[st.lid_off[type] + ser] = i;
  tgt_id[r] = i;
  tgt_time[r] = st.btime[slot];
  st.bstamp[slot] = -1;
  st.score[slot] = 0;
}

__global__ void k_sel_finish(hgt_gsample_state st, int32_t type, int64_t width, const unsigned long long* count,
                             int64_t* n_targets) {
  const int64_t m = (int64_t)*count < width ? (int64_t)*count : width;
  st.n_layer[type] += m;
  *n_targets = m;
}

// One warp per <block, target ser r>: neighbours of the target that are in the sample (data.py:190-209), counted, with
// the edge_time range check of to_torch (data.py:250; RelTemporalEncoding has 240 rows).
__global__ void k_rb_count(hgt_gsample_state st, const hgt_gsample_block* blocks, const int64_t* cnt_off, int64_t* cnt,
                           int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const hgt_gsample_block blk = blocks[b];
  const int T = blk.tgt_type, S = blk.src_type;
  if (r >= cnt_off[b + 1] - cnt_off[b]) return;
  int64_t c = 0;
  if (r < st.n_layer[T]) {
    const int64_t tid = st.lid[st.lid_off[T] + r];
    const int64_t row = tid < blk.n_row_of ? blk.row_of[tid] : -1;
    if (row >= 0) {
      const int64_t a = blk.ptr[row], e = blk.ptr[row + 1];
      const int64_t tt = st.ltime[st.type_off[T] + tid];
      const int64_t sb = st.type_off[S], sn = st.type_off[S + 1] - sb;
      for (int64_t p = a + lane; p < e; p += 32) {
        const int64_t sid = blk.nbr[p];
        if (sid < 0 || sid >= sn) { flags[0] = 1; continue; }
        if (st.ser[sb + sid] < 0) continue;
        ++c;
        const int64_t dt = tt - st.ltime[sb + sid] + 120;
        if (dt < 0 || dt >= HGT_RTE_MAX_LEN) flags[1] = 1;
      }
    }
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
  if (lane == 0) cnt[cnt_off[b] + r] = c;
}

__global__ void k_rb_totals(const int64_t* ex, const int64_t* cnt_off, int32_t n_blocks, int64_t* totals) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < n_blocks) totals[b] = ex[cnt_off[b + 1]] - ex[cnt_off[b]];
}

__global__ void k_rb_check_features(hgt_gsample_state st, const int64_t* feat_rows, int32_t* flags) {
  const int t = blockIdx.y;
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r < st.n_layer[t] && st.lid[st.lid_off[t] + r] >= feat_rows[t]) flags[2] = 1;
}

__global__ void k_rb_write(hgt_gsample_state st, const hgt_gsample_block* blocks, const int64_t* cnt_off,
                           const int64_t* ex, const int64_t* blk_out, const int64_t* node_off, int64_t n_edges,
                           int64_t* edge_index, int64_t* edge_type, int64_t* edge_time) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const hgt_gsample_block blk = blocks[b];
  const int T = blk.tgt_type, S = blk.src_type;
  if (blk_out[b] < 0 || r >= st.n_layer[T]) return;
  const int64_t tid = st.lid[st.lid_off[T] + r];
  const int64_t row = tid < blk.n_row_of ? blk.row_of[tid] : -1;
  if (row < 0) return;
  int64_t e = blk_out[b] + ex[cnt_off[b] + r] - ex[cnt_off[b]];
  const int64_t a = blk.ptr[row], end = blk.ptr[row + 1];
  const int64_t tt = st.ltime[st.type_off[T] + tid];
  const int64_t sb = st.type_off[S], sn = st.type_off[S + 1] - sb;
  const int64_t dst = node_off[T] + r;
  for (int64_t p0 = a; p0 < end; p0 += 32) {
    const int64_t p = p0 + lane;
    int32_t sser = -1;
    int64_t sid = -1;
    if (p < end) {
      sid = blk.nbr[p];
      if (sid >= 0 && sid < sn) sser = st.ser[sb + sid];
    }
    const unsigned keep = __ballot_sync(kFull, sser >= 0);
    if (sser >= 0) {
      const int64_t o = e + __popc(keep & ((1u << lane) - 1u));
      edge_index[o] = node_off[S] + sser;                               // row 0 = source (data.py:245,254)
      edge_index[n_edges + o] = dst;
      edge_type[o] = blk.rel;
      edge_time[o] = tt - st.ltime[sb + sid] + 120;                     // data.py:250
    }
    e += __popc(keep);
  }
}

// Nodes type by type (graph.get_types() order, ser order within a type: data.py:228-235), their self loops
// (data.py:181-184), and the feature rows gathered from the caller's per-type tables.
__global__ void k_rb_nodes(hgt_gsample_state st, const int64_t* node_off, const int64_t* type_out, const int64_t* self_off,
                           int64_t self_rel, int64_t n_edges, const float* const* feat, int32_t feat_dim,
                           int64_t* node_type, int64_t* node_time, float* node_feature, int64_t* edge_index,
                           int64_t* edge_type, int64_t* edge_time) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int t = blockIdx.y;
  if (node_off[t] < 0 || r >= st.n_layer[t]) return;
  const int64_t row = node_off[t] + r;
  const int64_t tid = st.lid[st.lid_off[t] + r];
  if (lane == 0) {
    node_type[row] = type_out[t];
    node_time[row] = st.ltime[st.type_off[t] + tid];
    if (self_off[t] >= 0) {
      const int64_t e = self_off[t] + r;
      edge_index[e] = row;
      edge_index[n_edges + e] = row;
      edge_type[e] = self_rel;
      edge_time[e] = 120;
    }
  }
  if (node_feature) {
    const float* src = feat[t] + tid * (int64_t)feat_dim;
    float* dst = node_feature + row * (int64_t)feat_dim;
    for (int c = lane; c < feat_dim; c += 32) dst[c] = src[c];
  }
}

struct BudgetScratch {
  int64_t *seg_cnt, *seg_off, *cand_pos, *cand_slot, *cand_time;
  void* cub_tmp;
  size_t cub_bytes;
};

size_t carve_budget(BudgetScratch& s, void* base, int64_t n_seg, int64_t cap) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += hgt_align_up(bytes, 256);
    return base ? (char*)base + o : (char*)nullptr;
  };
  s.seg_cnt = (int64_t*)take(sizeof(int64_t) * (n_seg + 1));
  s.seg_off = (int64_t*)take(sizeof(int64_t) * (n_seg + 1));
  s.cand_pos = (int64_t*)take(sizeof(int64_t) * (cap + 1));
  s.cand_slot = (int64_t*)take(sizeof(int64_t) * (cap + 1));
  s.cand_time = (int64_t*)take(sizeof(int64_t) * (cap + 1));
  s.cub_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, s.cub_bytes, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(n_seg + 1));
  s.cub_tmp = take(s.cub_bytes);
  return off;
}

struct SelectScratch {
  double *keys_in, *keys_out;
  int32_t *vals_in, *vals_out;
  unsigned long long* count;
  void* cub_tmp;
  size_t cub_bytes;
};

size_t carve_select(SelectScratch& s, void* base, int64_t n) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off += hgt_align_up(bytes, 256);
    return base ? (char*)base + o : (char*)nullptr;
  };
  s.keys_in = (double*)take(sizeof(double) * (n + 1));
  s.keys_out = (double*)take(sizeof(double) * (n + 1));
  s.vals_in = (int32_t*)take(sizeof(int32_t) * (n + 1));
  s.vals_out = (int32_t*)take(sizeof(int32_t) * (n + 1));
  s.count = (unsigned long long*)take(sizeof(unsigned long long));
  s.cub_bytes = 0;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, s.cub_bytes, (const double*)nullptr, (double*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1));
  s.cub_tmp = take(s.cub_bytes);
  return off;
}

inline int64_t blocks_for(int64_t n, int per = kThreads) { return (n + per - 1) / per; }

}  // namespace

extern "C" int hgt_gsample_add_budget_workspace_bytes(int64_t max_targets, int32_t n_blocks, int64_t sampled_number,
                                                      size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && max_targets >= 0 && n_blocks >= 0 && sampled_number > 0,
              "hgt_gsample_add_budget_workspace_bytes: bad arguments");
  const int64_t n_seg = max_targets * n_blocks;
  HGT_REQUIRE(n_seg < (int64_t(1) << 31) && n_seg * sampled_number < (int64_t(1) << 40),
              "hgt_gsample_add_budget_workspace_bytes: %lld targets x %d blocks x width %lld is too large",
              (long long)max_targets, n_blocks, (long long)sampled_number);
  BudgetScratch s;
  *out_bytes = carve_budget(s, nullptr, n_seg, n_seg * sampled_number);
  return 0;
}

extern "C" int hgt_gsample_add_budget(const hgt_gsample_state* h_state, const hgt_gsample_block* blocks,
                                      int32_t n_blocks, const int64_t* tgt_id, const int64_t* tgt_time,
                                      int64_t max_targets, const int64_t* n_targets, int64_t sampled_number,
                                      int32_t time_filter, int64_t max_time, int64_t no_time, uint64_t seed,
                                      int64_t step, int32_t* flags, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  HGT_REQUIRE(h_state && sampled_number > 0 && max_targets >= 0 && n_blocks >= 0 && step >= 0 && step < (1 << 22),
              "hgt_gsample_add_budget: bad arguments");
  const int64_t n_seg = max_targets * n_blocks;
  if (n_seg == 0) return 0;
  size_t need = 0;
  if (int rc = hgt_gsample_add_budget_workspace_bytes(max_targets, n_blocks, sampled_number, &need)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_gsample_add_budget: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cap = n_seg * sampled_number;
  BudgetScratch s;
  carve_budget(s, workspace, n_seg, cap);
  k_seg_count<<<blocks_for(n_seg + 1), kThreads, 0, st>>>(blocks, n_blocks, tgt_id, max_targets, n_targets,
                                                         sampled_number, s.seg_cnt);
  HGT_LAUNCH_CHECK();
  size_t tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(s.cub_tmp, tmp, s.seg_cnt, s.seg_off, (int)(n_seg + 1), st));
  k_candidates<<<blocks_for(n_seg, kWarps), kThreads, 0, st>>>(
      *h_state, blocks, n_blocks, tgt_id, tgt_time, max_targets, s.seg_cnt, s.seg_off, sampled_number, time_filter,
      max_time, no_time, seed, step, s.cand_pos, s.cand_slot, s.cand_time, flags);
  HGT_LAUNCH_CHECK();
  k_resolve<<<blocks_for(cap), kThreads, 0, st>>>(*h_state, s.seg_off, n_seg, cap, s.cand_slot, s.cand_time,
                                                  step << 40);
  HGT_LAUNCH_CHECK();
  k_touch<<<1, 1, 0, st>>>(*h_state);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_select_workspace_bytes(int64_t n_ids, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_ids >= 0 && n_ids < (int64_t(1) << 31) - 1,
              "hgt_gsample_select_workspace_bytes: %lld ids do not fit int32 sort values", (long long)n_ids);
  SelectScratch s;
  *out_bytes = carve_select(s, nullptr, n_ids);
  return 0;
}

extern "C" int hgt_gsample_select(const hgt_gsample_state* h_state, int32_t type, int64_t n_ids, int64_t sampled_number,
                                  uint64_t seed, int64_t step, int64_t* tgt_id, int64_t* tgt_time, int64_t* n_targets,
                                  int32_t* flags, void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && type >= 0 && type < h_state->num_types && sampled_number > 0 && step >= 0 && step < (1 << 22),
              "hgt_gsample_select: bad arguments");
  size_t need = 0;
  if (int rc = hgt_gsample_select_workspace_bytes(n_ids, &need)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_gsample_select: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  SelectScratch s;
  carve_select(s, workspace, n_ids);
  HGT_CHECK_CUDA(cudaMemsetAsync(s.count, 0, sizeof(unsigned long long), st));
  if (n_ids > 0) {
    const int64_t g = blocks_for(n_ids);
    k_sel_count<<<(unsigned)(g < 1024 ? g : 1024), kThreads, 0, st>>>(*h_state, type, s.count);
    HGT_LAUNCH_CHECK();
    k_sel_keys<<<g, kThreads, 0, st>>>(*h_state, type, sampled_number, s.count, seed, step, s.keys_in, s.vals_in);
    HGT_LAUNCH_CHECK();
    size_t tmp = s.cub_bytes;
    HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairsDescending(s.cub_tmp, tmp, s.keys_in, s.keys_out, s.vals_in,
                                                             s.vals_out, (int)n_ids, 0, 64, st));
    k_sel_take<<<blocks_for(sampled_number), kThreads, 0, st>>>(*h_state, type, sampled_number, s.count, s.vals_out,
                                                                tgt_id, tgt_time, flags);
    HGT_LAUNCH_CHECK();
  }
  k_sel_finish<<<1, 1, 0, st>>>(*h_state, type, sampled_number, s.count, n_targets);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_rebuild_workspace_bytes(int64_t n_count, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_count >= 0 && n_count < (int64_t(1) << 31) - 1,
              "hgt_gsample_rebuild_workspace_bytes: bad count %lld", (long long)n_count);
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(n_count + 1));
  *out_bytes = hgt_align_up(sizeof(int64_t) * (n_count + 1), 256) + b;
  return 0;
}

extern "C" int hgt_gsample_rebuild_count(const hgt_gsample_state* h_state, const hgt_gsample_block* blocks,
                                         int32_t n_blocks, const int64_t* cnt_off, int64_t n_count, int64_t max_rows,
                                         const int64_t* feat_rows, int64_t* ex, int64_t* totals, int32_t* flags,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && n_blocks >= 0 && n_blocks < 65536 && h_state->num_types < 65536 && max_rows >= 0,
              "hgt_gsample_rebuild_count: bad arguments");
  size_t need = 0;
  if (int rc = hgt_gsample_rebuild_workspace_bytes(n_count, &need)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "hgt_gsample_rebuild_count: workspace too small (%zu < %zu)",
              workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* cnt = (int64_t*)workspace;
  void* cub_tmp = (char*)workspace + hgt_align_up(sizeof(int64_t) * (n_count + 1), 256);
  size_t tmp = workspace_bytes - hgt_align_up(sizeof(int64_t) * (n_count + 1), 256);
  HGT_CHECK_CUDA(cudaMemsetAsync(cnt + n_count, 0, sizeof(int64_t), st));
  if (n_blocks > 0 && max_rows > 0) {
    k_rb_count<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_blocks), kThreads, 0, st>>>(*h_state, blocks, cnt_off,
                                                                                           cnt, flags);
    HGT_LAUNCH_CHECK();
  }
  HGT_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, tmp, cnt, ex, (int)(n_count + 1), st));
  if (n_blocks > 0) {
    k_rb_totals<<<blocks_for(n_blocks), kThreads, 0, st>>>(ex, cnt_off, n_blocks, totals);
    HGT_LAUNCH_CHECK();
  }
  if (feat_rows && max_rows > 0 && h_state->num_types > 0) {
    k_rb_check_features<<<dim3((unsigned)blocks_for(max_rows), h_state->num_types), kThreads, 0, st>>>(*h_state,
                                                                                                      feat_rows, flags);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int hgt_gsample_rebuild_write(const hgt_gsample_state* h_state, const hgt_gsample_block* blocks,
                                         int32_t n_blocks, const int64_t* cnt_off, const int64_t* ex,
                                         const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
                                         const int64_t* self_off, int64_t self_rel, int64_t max_rows, int64_t n_edges,
                                         const float* const* feat, int32_t feat_dim, int64_t* node_type,
                                         int64_t* node_time, float* node_feature, int64_t* edge_index,
                                         int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(h_state && n_blocks >= 0 && n_blocks < 65536 && h_state->num_types < 65536 && max_rows >= 0 &&
                  feat_dim >= 0 && (node_feature == nullptr || feat != nullptr),
              "hgt_gsample_rebuild_write: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (max_rows == 0) return 0;
  if (n_blocks > 0) {
    k_rb_write<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_blocks), kThreads, 0, st>>>(
        *h_state, blocks, cnt_off, ex, blk_out, node_off, n_edges, edge_index, edge_type, edge_time);
    HGT_LAUNCH_CHECK();
  }
  if (h_state->num_types > 0) {
    k_rb_nodes<<<dim3((unsigned)blocks_for(max_rows, kWarps), h_state->num_types), kThreads, 0, st>>>(
        *h_state, node_off, type_out, self_off, self_rel, n_edges, feat, feat_dim, node_type, node_time, node_feature,
        edge_index, edge_type, edge_time);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}
