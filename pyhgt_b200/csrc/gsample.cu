// HGSampling on the GPU (reference pyHGT/data.py:87-256: sample_subgraph + to_torch), the device path of
// pyhgt_b200/sampler.py:sample_subgraphs_cuda.  Draws from the same distribution as the host sampler (which replays numpy's
// stream bit for bit) with a counter-based RNG (Philox), so the result is a function of (seed, inputs) alone:
//   * add_budget (data.py:108-130) for a whole batch of targets: one warp per <target, block> segment draws the ordered
//     uniform subset (Floyd's set + Fisher-Yates order == permutation(n)[:k]) and applies the filters; the budget is
//     updated with order-independent atomics (fixed-point score, max / min of the candidate's position in the
//     reference's processing order for the last-writer time and the first-entry stamp), so it is bitwise repeatable;
//   * selection (data.py:150-165): Efraimidis-Spirakis keys log(u)/score^2 sorted with CUB (same ordered distribution as
//     np.random.choice(p, replace=False)), or the insertion stamp when the budget is smaller than the width;
//   * rebuild (data.py:181-209) + to_torch layout (data.py:226-256): count / scan / write per adjacency block, optionally
//     dropping edges by per-block minimum target / source sers (the OAG scripts' label-leak mask).
// Every stage runs B independent subgraphs ("members") at once: each member has its own rows of the state, its own seed
// and its own step numbers, and everything a member computes depends on its own rows alone, so member b of a batch is
// bitwise a batch of b alone with b's seed (sample_subgraph_cuda is such a batch of one).
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

// Member m's rows of the batch state (the dense per-slot arrays are shared: type_off / lid_off hold absolute positions).
struct Member {
  const int64_t *type_off, *lid_off;
  int64_t *n_layer, *type_min, *type_seq, *counters;
};

__device__ __forceinline__ Member member(const hgt_gsample_batch_state& st, int m) {
  const int T = st.num_types;
  return {st.type_off + (int64_t)m * (T + 1), st.lid_off + (int64_t)m * (T + 1), st.n_layer + (int64_t)m * T,
          st.type_min + (int64_t)m * 2 * T, st.type_seq + (int64_t)m * 2 * T, st.counters + 2 * m};
}

// ---- where a node's state lives ---------------------------------------------------------------------------------------
// The kernels shared by the two layouts are templates over the state struct; these overloads are the only place where
// the layouts differ.  Dense: node id of type t sits at slot type_off[t] + id of an id-range-sized array.  Hashed: it
// sits at the entry of its member's type-t region whose key is id, and its time is stored per ser (like lid).

struct HMember {
  const int64_t *type_off, *lid_off, *n_ids;                            // type_off: the region starts (ent_off)
  int64_t *n_layer, *type_min, *type_seq, *counters;
  unsigned long long* fill;
};

__device__ __forceinline__ HMember member(const hgt_gsample_hash_state& st, int m) {
  const int T = st.num_types;
  return {st.ent_off + (int64_t)m * (T + 1), st.lid_off + (int64_t)m * (T + 1), st.n_ids + (int64_t)m * T,
          st.n_layer + (int64_t)m * T, st.type_min + (int64_t)m * 2 * T, st.type_seq + (int64_t)m * 2 * T,
          st.counters + 2 * m, st.fill + (int64_t)m * T};
}

// A type of one member: its slots (base, n = the id range) or its region (base, room entries), id range n, lid start lt.
struct DenseIx {
  int64_t base, n;
};
struct HashIx {
  int64_t base, room, n, lt;
  unsigned long long* fill;
};

__device__ __forceinline__ DenseIx type_ix(const hgt_gsample_batch_state&, const Member& mb, int t) {
  const int64_t base = mb.type_off[t];
  return {base, mb.type_off[t + 1] - base};
}
__device__ __forceinline__ HashIx type_ix(const hgt_gsample_hash_state&, const HMember& mb, int t) {
  const int64_t base = mb.type_off[t];
  return {base, mb.type_off[t + 1] - base, mb.n_ids[t], mb.lid_off[t], mb.fill + t};
}

constexpr long long kEmptyKey = -1;

// First probe position of id in a region of `room` entries (splitmix64 finaliser, then a multiply-high).
__device__ __forceinline__ int64_t hash_home(int64_t id, int64_t room) {
  uint64_t x = (uint64_t)id + 0x9e3779b97f4a7c15ULL;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ULL;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return (int64_t)__umul64hi(x, (uint64_t)room);
}

// The entry of id, or -1 (not in the region).  Linear probing, each entry at most once.
__device__ __forceinline__ int64_t hash_find(const int64_t* key, const HashIx& ix, int64_t id) {
  int64_t j = hash_home(id, ix.room);
  for (int64_t q = 0; q < ix.room; ++q) {
    const int64_t k = key[ix.base + j];
    if (k == id) return ix.base + j;
    if (k == kEmptyKey) return -1;
    if (++j == ix.room) j = 0;
  }
  return -1;
}

// The entry of id, claimed with one compare-and-swap if it has none.  A claim past half the room, or a region with no
// free entry, raises the overflow flag (flags[3]); the latter also returns -1 (skip the candidate).
__device__ __forceinline__ int64_t hash_claim(int64_t* key, const HashIx& ix, int64_t id, int32_t* flags) {
  int64_t j = hash_home(id, ix.room);
  for (int64_t q = 0; q < ix.room; ++q) {
    unsigned long long* p = (unsigned long long*)(key + ix.base + j);
    long long k = *(volatile long long*)p;
    if (k == kEmptyKey) {
      k = (long long)atomicCAS(p, (unsigned long long)kEmptyKey, (unsigned long long)id);
      if (k == kEmptyKey) {
        if (2 * (atomicAdd(ix.fill, 1ULL) + 1) > (unsigned long long)ix.room) flags[3] = 1;
        return ix.base + j;
      }
    }
    if (k == id) return ix.base + j;
    if (++j == ix.room) j = 0;
  }
  flags[3] = 1;
  return -1;
}

// add_budget's slot of a candidate (false: skip it).
__device__ __forceinline__ bool budget_slot(const hgt_gsample_batch_state&, const DenseIx& ix, int64_t sid,
                                            int32_t*, int64_t* slot) {
  *slot = ix.base + sid;
  return true;
}
__device__ __forceinline__ bool budget_slot(const hgt_gsample_hash_state& st, const HashIx& ix, int64_t sid,
                                            int32_t* flags, int64_t* slot) {
  *slot = hash_claim(st.key, ix, sid, flags);
  return *slot >= 0;
}

// ser of id (in range) in the member's sample, -1 = not sampled.
__device__ __forceinline__ int32_t ser_of(const hgt_gsample_batch_state& st, const DenseIx& ix, int64_t sid) {
  return st.ser[ix.base + sid];
}
__device__ __forceinline__ int32_t ser_of(const hgt_gsample_hash_state& st, const HashIx& ix, int64_t sid) {
  const int64_t e = hash_find(st.key, ix, sid);
  return e >= 0 ? st.ser[e] : -1;
}

// Time of a sampled node of type t: id `id`, ser r.
__device__ __forceinline__ int64_t node_ltime(const hgt_gsample_batch_state& st, const Member& mb, int t, int64_t id,
                                             int64_t) {
  return st.ltime[mb.type_off[t] + id];
}
__device__ __forceinline__ int64_t node_ltime(const hgt_gsample_hash_state& st, const HMember& mb, int t, int64_t,
                                             int64_t r) {
  return st.ltime[mb.lid_off[t] + r];
}
// The same for a source looked up through its type's index.
__device__ __forceinline__ int64_t src_ltime(const hgt_gsample_batch_state& st, const DenseIx& ix, int64_t sid,
                                            int32_t) {
  return st.ltime[ix.base + sid];
}
__device__ __forceinline__ int64_t src_ltime(const hgt_gsample_hash_state& st, const HashIx& ix, int64_t,
                                            int32_t sser) {
  return st.ltime[ix.lt + sser];
}

// The blocks member m's add_budget walks: those of the member's current type (type_blocks [2T]: begin / end per target
// type; type[m] < 0 = the member sits this step out).
struct BlockRange {
  const int32_t* type_blocks;
  const int32_t* type;
  __device__ __forceinline__ void get(int m, int32_t* b0, int32_t* nb) const {
    const int t = type[m];
    *b0 = 0;
    *nb = 0;
    if (t >= 0) {
      *b0 = type_blocks[2 * t];
      *nb = type_blocks[2 * t + 1] - *b0;
    }
  }
};

// Where member m's nodes and edges go in the output buffers: {node_base, edge_base, src_pos, dst_pos} per member: its
// edge e has edge_type / edge_time at edge_base + e and its endpoints at edge_index[src_pos + e] / [dst_pos + e].  Read-only
// loads: with plain ones the hashed k_rb_write takes 52 registers instead of 48 (sm_90a, CUDA 12.9).
struct MemOut {
  const int64_t* p;
  __device__ __forceinline__ int64_t node_base(int m) const { return __ldg(p + 4 * m); }
  __device__ __forceinline__ int64_t edge_base(int m) const { return __ldg(p + 4 * m + 1); }
  __device__ __forceinline__ int64_t src_pos(int m) const { return __ldg(p + 4 * m + 2); }
  __device__ __forceinline__ int64_t dst_pos(int m) const { return __ldg(p + 4 * m + 3); }
};

__device__ __forceinline__ uint64_t rnd64(curandStatePhilox4_32_10_t* s) {
  const uint64_t hi = curand(s);
  return (hi << 32) | curand(s);
}
// uniform in [0, m): multiply-high of a 64-bit draw (bias below m / 2^64)
__device__ __forceinline__ int64_t rnd_below(curandStatePhilox4_32_10_t* s, int64_t m) {
  return (int64_t)__umul64hi(rnd64(s), (uint64_t)m);
}

// ---- a block's arrays at either width ---------------------------------------------------------------------------------
// Every kernel reads row_of / ptr / nbr / time through these.  A narrow block (skip & HGT_BLOCK_NARROW) holds them as
// int32, with INT32_MIN for no_time.  A warp's segment or target row lies in one block, so the branch is warp-uniform.
__device__ __forceinline__ bool blk_narrow(const hgt_gsample_block& b) { return b.skip & HGT_BLOCK_NARROW; }
__device__ __forceinline__ int64_t blk_row(const hgt_gsample_block& b, int64_t tid) {
  return blk_narrow(b) ? (int64_t)reinterpret_cast<const int32_t*>(b.row_of)[tid] : b.row_of[tid];
}
__device__ __forceinline__ int64_t blk_ptr(const hgt_gsample_block& b, int64_t row) {
  return blk_narrow(b) ? (int64_t)reinterpret_cast<const int32_t*>(b.ptr)[row] : b.ptr[row];
}
__device__ __forceinline__ int64_t blk_nbr(const hgt_gsample_block& b, int64_t p) {
  return blk_narrow(b) ? (int64_t)reinterpret_cast<const int32_t*>(b.nbr)[p] : b.nbr[p];
}
__device__ __forceinline__ int64_t blk_time(const hgt_gsample_block& b, int64_t p, int64_t no_time) {
  if (!blk_narrow(b)) return b.time[p];
  const int32_t t = reinterpret_cast<const int32_t*>(b.time)[p];
  return t == INT32_MIN ? no_time : (int64_t)t;
}
// CSR row of target tid (-1: none); the neighbours of row are [blk_ptr(row), blk_ptr(row + 1)).
__device__ __forceinline__ int64_t blk_row_of(const hgt_gsample_block& b, int64_t tid) {
  return tid >= 0 && tid < b.n_row_of ? blk_row(b, tid) : -1;
}

__device__ __forceinline__ int64_t seg_size(const hgt_gsample_block& blk, int64_t tid, int64_t width, int64_t* a,
                                            int64_t* deg) {
  *a = 0;
  *deg = 0;
  if (blk.skip & HGT_BLOCK_SKIP) return 0;                              // 'self' (data.py:116)
  const int64_t row = blk_row_of(blk, tid);
  if (row < 0) return 0;                                                // no adjacency
  *a = blk_ptr(blk, row);
  *deg = blk_ptr(blk, row + 1) - *a;
  return *deg < width ? *deg : width;                                   // data.py:119-122
}

// Segments are member-major with stride S = max_targets * max_blocks; inside a member, segment k * nb + b is target k,
// block b (nb = the member's block count), the numbering of a batch of that member alone.
__global__ void k_seg_count(const hgt_gsample_block* blocks, BlockRange br, int32_t n_members, int64_t S,
                            const int64_t* tgt_id, int64_t max_targets, const int64_t* n_targets, int64_t width,
                            int64_t* seg_cnt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t n_seg = S * n_members;
  if (i > n_seg) return;
  if (i == n_seg) { seg_cnt[i] = 0; return; }
  const int m = (int)(i / S);
  const int64_t loc = i % S;
  int32_t b0, nb;
  br.get(m, &b0, &nb);
  int64_t c = 0;
  if (loc < max_targets * nb) {
    const int64_t k = loc / nb;
    int64_t a, deg;
    if (k < n_targets[m]) c = seg_size(blocks[b0 + loc % nb], tgt_id[m * max_targets + k], width, &a, &deg);
  }
  seg_cnt[i] = c;
}

// One warp per <member, target k, block b>.  seq = seg_off + j orders the member's candidates like the reference's
// processing order (target, block, neighbour in subset order), the key of every order-dependent rule.
template <class St>
__global__ void k_candidates(St st, const int64_t* step, const hgt_gsample_block* blocks, BlockRange br, int64_t S,
                             const int64_t* tgt_id, const int64_t* tgt_time, int64_t max_targets,
                             const int64_t* seg_cnt, const int64_t* seg_off, int64_t width, int32_t time_filter,
                             int64_t max_time, int64_t no_time, int64_t* cand_pos, int64_t* cand_slot,
                             int64_t* cand_time, int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (seg >= S * st.n_members) return;
  const int64_t n_s = seg_cnt[seg];
  if (n_s == 0) return;
  const int m = (int)(seg / S);
  const int64_t loc = seg % S;
  int32_t b0, nb;
  br.get(m, &b0, &nb);
  const auto mb = member(st, m);
  const int64_t k = loc / nb;
  const hgt_gsample_block blk = blocks[b0 + loc % nb];
  int64_t a, deg;
  seg_size(blk, tgt_id[m * max_targets + k], width, &a, &deg);
  const int64_t off = seg_off[seg];
  int64_t* S_ = cand_pos + off;
  const bool all = deg < width;
  if (!all) {
    // Floyd: a uniform n_s-subset of [0, deg); then a uniform order (Fisher-Yates).  Every lane runs the same stream.
    curandStatePhilox4_32_10_t rs;
    curand_init(st.seed[m], ((uint64_t)step[m] << 32) | (uint64_t)loc, 0, &rs);
    for (int64_t c = 0, jj = deg - n_s; jj < deg; ++jj, ++c) {
      const int64_t t = rnd_below(&rs, jj + 1);
      bool found = false;
      for (int64_t q = lane; q < c; q += 32) found |= (S_[q] == t);
      found = __any_sync(kFull, found);
      if (lane == 0) S_[c] = found ? jj : t;
      __syncwarp();
    }
    if (lane == 0)
      for (int64_t i = n_s - 1; i > 0; --i) {
        const int64_t j = rnd_below(&rs, i + 1);
        const int64_t x = S_[i];
        S_[i] = S_[j];
        S_[j] = x;
      }
    __syncwarp();
  }
  const int64_t target_time = tgt_time[m * max_targets + k];
  const int src = blk.src_type;
  const auto ix = type_ix(st, mb, src);
  const unsigned long long w = (unsigned long long)llrint(kScoreScale / (double)n_s);   // 1. / len(sampled_ids)
  for (int64_t j = lane; j < n_s; j += 32) {
    const int64_t seq = off + j;
    const int64_t pos = a + (all ? j : S_[j]);
    const int64_t sid = blk_nbr(blk, pos);
    int64_t tm = blk_time(blk, pos, no_time);
    if (tm == no_time) tm = target_time;                                // data.py:125-126
    cand_slot[seq] = -1;
    if (time_filter && tm > max_time) continue;                         // data.py:127, first operand of the `or`
    atomicMin((long long*)&mb.type_min[2 * src], (long long)seq);      // layer_data[source_type] springs into being
    if (sid < 0 || sid >= ix.n) { flags[0] = 1; continue; }
    int64_t slot;
    if (!budget_slot(st, ix, sid, flags, &slot)) continue;
    if (st.ser[slot] >= 0) continue;                                    // already sampled
    atomicMin((long long*)&mb.type_min[2 * src + 1], (long long)seq);  // budget[source_type] springs into being
    atomicAdd(&st.score[slot], w);
    atomicMax((long long*)&st.last_seq[slot], (long long)seq);
    if (st.bstamp[slot] < 0) atomicMin((long long*)&st.first_seq[slot], (long long)seq);
    cand_slot[seq] = slot;
    cand_time[seq] = tm;
  }
}

// The candidate that wrote last sets the budget time (data.py:130); the first one of a new entry sets its stamp (step
// << 40 + its position among the member's candidates).  The matching candidate also resets the scratch word: no other
// candidate of the slot can match either value.  grid.y = member; grid-stride over the member's candidates.
template <class St>
__global__ void k_resolve(St st, const int64_t* step, const int64_t* seg_off, int64_t S,
                          const int64_t* cand_slot, const int64_t* cand_time) {
  const int m = blockIdx.y;
  const int64_t lo = seg_off[m * S], hi = seg_off[(m + 1) * S];
  const int64_t stamp_base = step[m] << 40;
  for (int64_t seq = lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; seq < hi;
       seq += (int64_t)gridDim.x * blockDim.x) {
    const int64_t slot = cand_slot[seq];
    if (slot < 0) continue;
    if (st.last_seq[slot] == seq) {
      st.btime[slot] = cand_time[seq];
      st.last_seq[slot] = -1;
    }
    if (st.first_seq[slot] == seq) {
      st.bstamp[slot] = stamp_base + (seq - lo);
      st.first_seq[slot] = kNoSeq;
    }
  }
}

// First-touch numbers of layer_data[t] / budget[t] (the key orders of the reference's defaultdicts): types touched for
// the first time in this step are numbered in the order of their first qualifying candidate.  One thread per member.
template <class St>
__global__ void k_touch(St st) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= st.n_members) return;
  const auto mb = member(st, m);
  for (int kind = 0; kind < 2; ++kind) {
    for (;;) {
      int best = -1;
      long long bv = kNoSeq;
      for (int t = 0; t < st.num_types; ++t)
        if (mb.type_seq[2 * t + kind] < 0 && mb.type_min[2 * t + kind] < bv) { bv = mb.type_min[2 * t + kind]; best = t; }
      if (best < 0) break;
      mb.type_seq[2 * best + kind] = mb.counters[kind]++;
    }
    for (int t = 0; t < st.num_types; ++t) mb.type_min[2 * t + kind] = kNoSeq;
  }
}

// grid.y = member, which selects from its own type[m] (< 0: none this step).
__global__ void k_sel_count(hgt_gsample_batch_state st, const int32_t* type, unsigned long long* count) {
  const int m = blockIdx.y;
  const int t = type[m];
  if (t < 0) return;
  const Member mb = member(st, m);
  const int64_t base = mb.type_off[t], n = mb.type_off[t + 1] - base;
  unsigned long long c = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    c += st.bstamp[base + i] >= 0;
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&count[m], c);
}

// Sort keys (descending): budget smaller than the width -> every entry in insertion order (key -stamp); otherwise
// Efraimidis-Spirakis log(u) / score^2 (data.py:158-160).  Entries outside the budget sort last.  Member m's ids sit at
// sel_off[m] + i; the sort value is that position.
__global__ void k_sel_keys(hgt_gsample_batch_state st, const int32_t* type, const int64_t* sel_off, int64_t width,
                           const unsigned long long* count, const int64_t* step, double* keys, int32_t* vals) {
  const int m = blockIdx.y;
  const int t = type[m];
  if (t < 0) return;
  const Member mb = member(st, m);
  const int64_t base = mb.type_off[t], n = mb.type_off[t + 1] - base;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t slot = base + i;
  const int64_t stamp = st.bstamp[slot];
  double key = -INFINITY;
  if (stamp >= 0) {
    if (width > (int64_t)count[m]) {
      key = -(double)stamp;
    } else {
      curandStatePhilox4_32_10_t rs;
      curand_init(st.seed[m] ^ kSelectStream, ((uint64_t)step[m] << 40) | (uint64_t)i, 0, &rs);
      const double u = (double)((rnd64(&rs) >> 11) + 1) * 0x1.0p-53;   // (0, 1]
      const double s = (double)st.score[slot] / kScoreScale;
      key = log(u) / (s * s);
    }
  }
  const int64_t o = sel_off[m] + i;
  keys[o] = key;
  vals[o] = (int32_t)o;
}

// Second, stable pass of the batched sort: the member of every sorted entry (the last m with sel_off[m] <= position),
// so that sorting by it keeps each member's entries together in key order.
__global__ void k_sel_member(const int64_t* sel_off, int32_t n_members, const int32_t* vals, int64_t n, int32_t* mkey) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t v = vals[j];
  int lo = 0, hi = n_members;                                           // sel_off[lo] <= v < sel_off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sel_off[mid] <= v) lo = mid; else hi = mid;
  }
  mkey[j] = lo;
}

// data.py:166-170: the chosen ids join layer_data in key order (ser), become the next add_budget's targets (member m's
// at tgt_id[m * width ...]), and leave the budget.
__global__ void k_sel_take(hgt_gsample_batch_state st, const int32_t* type, const int64_t* sel_off, int64_t width,
                           const unsigned long long* count, const int32_t* vals, int64_t* tgt_id, int64_t* tgt_time,
                           int32_t* flags) {
  const int m = blockIdx.y;
  const int t = type[m];
  if (t < 0) return;
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = (int64_t)count[m] < width ? (int64_t)count[m] : width;
  if (r >= c) return;
  const Member mb = member(st, m);
  const int64_t o = sel_off[m];
  const int64_t i = vals[o + r] - o;
  const int64_t slot = mb.type_off[t] + i;
  const int64_t ser = mb.n_layer[t] + r;
  if (mb.lid_off[t] + ser >= mb.lid_off[t + 1]) { flags[0] = 1; return; }
  st.ser[slot] = (int32_t)ser;
  st.ltime[slot] = st.btime[slot];
  st.lid[mb.lid_off[t] + ser] = i;
  tgt_id[m * width + r] = i;
  tgt_time[m * width + r] = st.btime[slot];
  st.bstamp[slot] = -1;
  st.score[slot] = 0;
}

template <class St>
__global__ void k_sel_finish(St st, const int32_t* type, int64_t width, const unsigned long long* count,
                             int64_t* n_targets) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= st.n_members) return;
  const int t = type[m];
  if (t < 0) { n_targets[m] = 0; return; }
  const int64_t c = (int64_t)count[m] < width ? (int64_t)count[m] : width;
  member(st, m).n_layer[t] += c;
  n_targets[m] = c;
}

// ---- the hashed state's own kernels: seeds and selection ------------------------------------------------------------

// Seed i: an entry for id[i] in region[i] = m * T + t with its ser, and lid / ltime at that ser (region[i] < 0: none).
__global__ void k_hash_seed(hgt_gsample_hash_state st, int64_t n, const int64_t* region, const int64_t* id,
                            const int64_t* ser, const int64_t* time, int32_t* flags) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n || region[i] < 0) return;
  const int m = (int)(region[i] / st.num_types), t = (int)(region[i] % st.num_types);
  const HMember mb = member(st, m);
  const HashIx ix = type_ix(st, mb, t);
  const int64_t e = hash_claim(st.key, ix, id[i], flags);
  if (e < 0) return;
  st.ser[e] = (int32_t)ser[i];
  st.lid[mb.lid_off[t] + ser[i]] = id[i];
  st.ltime[mb.lid_off[t] + ser[i]] = time[i];
}

constexpr int kIdBits = 41;                                             // ids < 2^40, plus "not in the budget"
constexpr uint64_t kNotBudget = (uint64_t(1) << kIdBits) - 1;

// A sort of n_total >= sel_off[B] positions (the caller's upper bound when the regions are chosen on the device): the
// positions past sel_off[B] are padding, max_room - (member m's region size) of them per member, member after member.
// Position of member m's padding j, or -1 when it lies past n_total (always so when n_total = sel_off[B]).
__device__ __forceinline__ int64_t sel_pad_pos(const int64_t* sel_off, int B, int m, int64_t max_room, int64_t n_total,
                                               int64_t j) {
  const int64_t p = sel_off[B] + m * max_room - sel_off[m] + j;
  return p < n_total ? p : -1;
}

// Selection pass 1: every entry of member m's region of type[m], at sel_off[m] + its index, gets the sort key
// (m, id) when it is in the budget and (m, kNotBudget) otherwise, so that sorting puts each member's budget entries
// first and in id order: the order of the dense selection's positions.  Counts the budget entries.  Padding positions
// take the largest key, so they sort behind every member's entries.
__global__ void k_hsel_order(hgt_gsample_hash_state st, const int32_t* type, const int64_t* sel_off, int64_t max_room,
                             int64_t n_total, uint64_t* okey, int64_t* oent, unsigned long long* count) {
  const int m = blockIdx.y;
  const int t = type[m];
  const HMember mb = member(st, m);
  const int64_t base = t >= 0 ? mb.type_off[t] : 0, n = t >= 0 ? mb.type_off[t + 1] - base : 0, o = sel_off[m];
  unsigned long long c = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < max_room; i += (int64_t)gridDim.x * blockDim.x) {
    if (i >= n) {
      const int64_t p = sel_pad_pos(sel_off, st.n_members, m, max_room, n_total, i - n);
      if (p >= 0) {
        okey[p] = ~0ULL;
        oent[p] = -1;
      }
      continue;
    }
    const bool in = st.bstamp[base + i] >= 0;
    okey[o + i] = ((uint64_t)m << kIdBits) | (in ? (uint64_t)st.key[base + i] : kNotBudget);
    oent[o + i] = base + i;
    c += in;
  }
  for (int s = 16; s; s >>= 1) c += __shfl_xor_sync(kFull, c, s);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&count[m], c);
}

// k_sel_keys over the id-ordered entries: the first count[m] positions of member m are its budget, the node id is the
// Philox counter's local id, so every key is bitwise the dense one.
// Padding positions get key -inf, behind every budget key.
__global__ void k_hsel_keys(hgt_gsample_hash_state st, const int32_t* type, const int64_t* sel_off, int64_t max_room,
                            int64_t n_total, int64_t width, const unsigned long long* count, const int64_t* step,
                            const uint64_t* okey, const int64_t* oent, double* keys, int32_t* vals) {
  const int m = blockIdx.y;
  const int t = type[m];
  const HMember mb = member(st, m);
  const int64_t n = t >= 0 ? mb.type_off[t + 1] - mb.type_off[t] : 0;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) {
    const int64_t p = i < max_room ? sel_pad_pos(sel_off, st.n_members, m, max_room, n_total, i - n) : -1;
    if (p >= 0) {
      keys[p] = -INFINITY;
      vals[p] = (int32_t)p;
    }
    return;
  }
  const int64_t o = sel_off[m] + i;
  double key = -INFINITY;
  if (i < (int64_t)count[m]) {
    const int64_t e = oent[o];
    if (width > (int64_t)count[m]) {
      key = -(double)st.bstamp[e];
    } else {
      const uint64_t id = okey[o] & kNotBudget;
      curandStatePhilox4_32_10_t rs;
      curand_init(st.seed[m] ^ kSelectStream, ((uint64_t)step[m] << 40) | id, 0, &rs);
      const double u = (double)((rnd64(&rs) >> 11) + 1) * 0x1.0p-53;   // (0, 1]
      const double s = (double)st.score[e] / kScoreScale;
      key = log(u) / (s * s);
    }
  }
  keys[o] = key;
  vals[o] = (int32_t)o;
}

// k_sel_take with the chosen entry found through the id order.
__global__ void k_hsel_take(hgt_gsample_hash_state st, const int32_t* type, const int64_t* sel_off, int64_t width,
                            const unsigned long long* count, const int32_t* vals, const int64_t* oent, int64_t* tgt_id,
                            int64_t* tgt_time, int32_t* flags) {
  const int m = blockIdx.y;
  const int t = type[m];
  if (t < 0) return;
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = (int64_t)count[m] < width ? (int64_t)count[m] : width;
  if (r >= c) return;
  const HMember mb = member(st, m);
  const int64_t e = oent[vals[sel_off[m] + r]];
  const int64_t id = st.key[e];
  const int64_t ser = mb.n_layer[t] + r;
  const int64_t l = mb.lid_off[t] + ser;
  if (l >= mb.lid_off[t + 1]) { flags[0] = 1; return; }
  st.ser[e] = (int32_t)ser;
  st.ltime[l] = st.btime[e];
  st.lid[l] = id;
  tgt_id[m * width + r] = id;
  tgt_time[m * width + r] = st.btime[e];
  st.bstamp[e] = -1;
  st.score[e] = 0;
}

// The caller's edge mask (sampler.py: edge_mask; the OAG scripts drop the edges that would leak a seed's label between
// sample_subgraph and to_torch): an edge of block b with target ser r and source ser sser is dropped unless
// r >= min_ser[2b] and sser >= min_ser[2b+1].  min_ser == NULL keeps every edge.  Both rebuild passes use this one
// predicate, so the count pass's prefix sum and the edges the write pass lays out agree.
__device__ __forceinline__ bool masked_out(const int64_t* min_ser, int b, int64_t r, int64_t sser) {
  return min_ser && (r < min_ser[2 * b] || sser < min_ser[2 * b + 1]);
}

// One warp per <member (grid.z), block (grid.y), target ser r>: neighbours of the target that are in the member's sample
// (data.py:190-209) and not masked out, counted, with the edge_time range check of to_torch on those kept edges
// (data.py:250; RelTemporalEncoding has 240 rows).
template <class St>
__global__ void k_rb_count(St st, const hgt_gsample_block* blocks, int32_t n_blocks,
                           const int64_t* min_ser, const int64_t* cnt_off, int64_t* cnt, int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const int64_t mbk = (int64_t)blockIdx.z * n_blocks + b;
  const hgt_gsample_block blk = blocks[b];
  const int T = blk.tgt_type, S = blk.src_type;
  if (r >= cnt_off[mbk + 1] - cnt_off[mbk]) return;
  const auto mb = member(st, blockIdx.z);
  int64_t c = 0;
  if (r < mb.n_layer[T]) {
    const int64_t tid = st.lid[mb.lid_off[T] + r];
    const int64_t row = blk_row_of(blk, tid);
    if (row >= 0) {
      const int64_t a = blk_ptr(blk, row), e = blk_ptr(blk, row + 1);
      const int64_t tt = node_ltime(st, mb, T, tid, r);
      const auto ix = type_ix(st, mb, S);
      for (int64_t p = a + lane; p < e; p += 32) {
        const int64_t sid = blk_nbr(blk, p);
        if (sid < 0 || sid >= ix.n) { flags[0] = 1; continue; }
        const int32_t sser = ser_of(st, ix, sid);
        if (sser < 0 || masked_out(min_ser, b, r, sser)) continue;
        ++c;
        const int64_t dt = tt - src_ltime(st, ix, sid, sser) + 120;
        if (dt < 0 || dt >= HGT_RTE_MAX_LEN) flags[1] = 1;
      }
    }
  }
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
  if (lane == 0) cnt[cnt_off[mbk] + r] = c;
}

__global__ void k_rb_totals(const int64_t* ex, const int64_t* cnt_off, int64_t n, int64_t* totals) {
  const int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (b < n) totals[b] = ex[cnt_off[b + 1]] - ex[cnt_off[b]];
}

template <class St>
__global__ void k_rb_check_features(St st, const int64_t* feat_rows, int32_t* flags) {
  const int t = blockIdx.y;
  const auto mb = member(st, blockIdx.z);
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r < mb.n_layer[t] && st.lid[mb.lid_off[t] + r] >= feat_rows[t]) flags[2] = 1;
}

// blk_out / node_off / self_off are member-local (member m's rows [m * n_blocks ...] / [m * T ...]); edge_index holds
// each member's [2, E_m] block at 2 * edge_base, node ids member-local.  The ballot keeps the kept edges in block order.
template <class St>
__global__ void k_rb_write(St st, const hgt_gsample_block* blocks, int32_t n_blocks,
                           const int64_t* min_ser, const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out,
                           const int64_t* node_off, MemOut mo, int64_t* edge_index, int64_t* edge_type,
                           int64_t* edge_time) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const int m = blockIdx.z;
  const int64_t mbk = (int64_t)m * n_blocks + b;
  const hgt_gsample_block blk = blocks[b];
  const int T = blk.tgt_type, S = blk.src_type;
  const auto mb = member(st, m);
  if (blk_out[mbk] < 0 || r >= mb.n_layer[T]) return;
  const int64_t tid = st.lid[mb.lid_off[T] + r];
  const int64_t row = blk_row_of(blk, tid);
  if (row < 0) return;
  const int64_t* noff = node_off + (int64_t)m * st.num_types;
  const int64_t eb = mo.edge_base(m);
  int64_t* ei_src = edge_index + mo.src_pos(m);
  int64_t* ei_dst = edge_index + mo.dst_pos(m);
  int64_t e = blk_out[mbk] + ex[cnt_off[mbk] + r] - ex[cnt_off[mbk]];
  const int64_t a = blk_ptr(blk, row), end = blk_ptr(blk, row + 1);
  const int64_t tt = node_ltime(st, mb, T, tid, r);
  const auto ix = type_ix(st, mb, S);
  const int64_t dst = noff[T] + r;
  for (int64_t p0 = a; p0 < end; p0 += 32) {
    const int64_t p = p0 + lane;
    int32_t sser = -1;
    int64_t sid = -1;
    if (p < end) {
      sid = blk_nbr(blk, p);
      if (sid >= 0 && sid < ix.n) sser = ser_of(st, ix, sid);
    }
    const bool kept = sser >= 0 && !masked_out(min_ser, b, r, sser);
    const unsigned keep = __ballot_sync(kFull, kept);
    if (kept) {
      const int64_t o = e + __popc(keep & ((1u << lane) - 1u));
      ei_src[o] = noff[S] + sser;                                       // row 0 = source (data.py:245,254)
      ei_dst[o] = dst;
      edge_type[eb + o] = blk.rel;
      edge_time[eb + o] = tt - src_ltime(st, ix, sid, sser) + 120;        // data.py:250
    }
    e += __popc(keep);
  }
}

// Nodes type by type (graph.get_types() order, ser order within a type: data.py:228-235), their self loops
// (data.py:181-184), and the feature rows gathered from the caller's per-type tables.  grid.z = member.
template <class St>
__global__ void k_rb_nodes(St st, const int64_t* node_off, const int64_t* type_out,
                           const int64_t* self_off, int64_t self_rel, MemOut mo, const float* const* feat,
                           int32_t feat_dim, int64_t* node_type, int64_t* node_time, float* node_feature,
                           int64_t* edge_index, int64_t* edge_type, int64_t* edge_time) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int t = blockIdx.y;
  const int m = blockIdx.z;
  const auto mb = member(st, m);
  const int64_t noff = node_off[(int64_t)m * st.num_types + t];
  if (noff < 0 || r >= mb.n_layer[t]) return;
  const int64_t lrow = noff + r;
  const int64_t row = mo.node_base(m) + lrow;
  const int64_t tid = st.lid[mb.lid_off[t] + r];
  if (lane == 0) {
    node_type[row] = type_out[t];
    node_time[row] = node_ltime(st, mb, t, tid, r);
    const int64_t so = self_off[(int64_t)m * st.num_types + t];
    if (so >= 0) {
      const int64_t e = so + r, eb = mo.edge_base(m);
      edge_index[mo.src_pos(m) + e] = lrow;
      edge_index[mo.dst_pos(m) + e] = lrow;
      edge_type[eb + e] = self_rel;
      edge_time[eb + e] = 120;
    }
  }
  if (node_feature) {
    const float* src = feat[t] + tid * (int64_t)feat_dim;
    float* dst = node_feature + row * (int64_t)feat_dim;
    for (int c = lane; c < feat_dim; c += 32) dst[c] = src[c];
  }
}

// ---- graphs in page-locked host memory (sampler.py: DeviceGraph(..., placement="host")) ------------------------------
// The kernels above read row_of / ptr / nbr / time and the feature tables in place wherever they live, so add_budget's
// random neighbour draws run unchanged on a host-resident graph.  The rebuild gets its own instances: over PCIe, reading
// every sampled target's neighbour list twice (count pass, then write pass) doubles the dominant traffic, and 4-byte
// feature copies leave the link idle.  The count pass below reads each list once and leaves one hit record per kept edge
// in device scratch; the write pass lays the edges out from those records alone.

constexpr int kListUnroll = 8;   // neighbour ids in flight per lane in the single-read count pass (16 for int32 lists:
                                 // the same 64 bytes per lane)
constexpr int kRowUnroll = 4;    // 16-byte feature loads in flight per lane in the host gather

// A kept edge: {m * n_blocks + b, target ser r, rank among r's kept edges in list order, source ser}.  Its output position
// is blk_out + (ex[r] - ex[0]) + rank, so the records may sit in the scratch in any order.
using Hit = int4;

// The list [a, e) of nbr (Id = the block's element type) in chunks of 32 * U ids, U loads in flight per lane: counts,
// flags and hit records of k_rb_count_host.  Returns the number of kept edges.
template <int U, typename Id, class St, class Ix>
__device__ __forceinline__ int64_t count_list_host(const St& st, const Ix& ix, const Id* nbr, int64_t a, int64_t e,
                                                   int64_t tt, const int64_t* min_ser, int b, int64_t r, int64_t mbk,
                                                   Hit* hits, int64_t hit_cap, unsigned long long* n_hits,
                                                   int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  int64_t c = 0;                                                        // kept edges so far (warp-uniform)
  for (int64_t p0 = a; p0 < e; p0 += 32 * U) {
    int64_t sid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t p = p0 + 32 * u + lane;
      sid[u] = p < e ? (int64_t)nbr[p] : -1;
    }
    int32_t sser[U];
    unsigned keep[U];
    int n_kept = 0;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t p = p0 + 32 * u + lane;
      sser[u] = -1;
      if (p < e) {
        if (sid[u] < 0 || sid[u] >= ix.n) flags[0] = 1;
        else sser[u] = ser_of(st, ix, sid[u]);
      }
      const bool kept = sser[u] >= 0 && !masked_out(min_ser, b, r, sser[u]);
      if (kept) {
        const int64_t dt = tt - src_ltime(st, ix, sid[u], sser[u]) + 120;
        if (dt < 0 || dt >= HGT_RTE_MAX_LEN) flags[1] = 1;
      }
      keep[u] = __ballot_sync(kFull, kept);
      n_kept += __popc(keep[u]);
    }
    if (n_kept == 0) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(n_hits, (unsigned long long)n_kept);
    base = __shfl_sync(kFull, base, 0);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int k = __popc(keep[u] & below);
      if ((keep[u] >> lane) & 1u && (int64_t)base + k < hit_cap)
        hits[base + k] = make_int4((int)mbk, (int)r, (int)(c + k), sser[u]);
      base += __popc(keep[u]);
      c += __popc(keep[u]);
    }
  }
  return c;
}

// k_rb_count's counts, flags and mask, plus the hit records: slots claimed with one atomic per warp and one chunk of
// neighbours; records past hit_cap are dropped (n_hits still counts them, so the caller sees the overflow).
template <class St>
__global__ void k_rb_count_host(St st, const hgt_gsample_block* blocks, int32_t n_blocks,
                                const int64_t* min_ser, const int64_t* cnt_off, int64_t* cnt, Hit* hits,
                                int64_t hit_cap, unsigned long long* n_hits, int32_t* flags) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int b = blockIdx.y;
  const int64_t mbk = (int64_t)blockIdx.z * n_blocks + b;
  const hgt_gsample_block blk = blocks[b];
  const int T = blk.tgt_type, S = blk.src_type;
  if (r >= cnt_off[mbk + 1] - cnt_off[mbk]) return;
  const auto mb = member(st, blockIdx.z);
  int64_t c = 0;
  if (r < mb.n_layer[T]) {
    const int64_t tid = st.lid[mb.lid_off[T] + r];
    const int64_t row = blk_row_of(blk, tid);
    if (row >= 0) {
      const int64_t a = blk_ptr(blk, row), e = blk_ptr(blk, row + 1);
      const int64_t tt = node_ltime(st, mb, T, tid, r);
      const auto ix = type_ix(st, mb, S);
      if (blk_narrow(blk))
        c = count_list_host<2 * kListUnroll>(st, ix, reinterpret_cast<const int32_t*>(blk.nbr), a, e, tt, min_ser, b,
                                             r, mbk, hits, hit_cap, n_hits, flags);
      else
        c = count_list_host<kListUnroll>(st, ix, blk.nbr, a, e, tt, min_ser, b, r, mbk, hits, hit_cap, n_hits, flags);
    }
  }
  if (lane == 0) cnt[cnt_off[mbk] + r] = c;
}

// One thread per hit record: k_rb_write's outputs without touching the graph (the source id and both times come from
// the member's device state).
template <class St>
__global__ void k_rb_write_hits(St st, const hgt_gsample_block* blocks, int32_t n_blocks,
                                const Hit* hits, int64_t n_hits, const int64_t* cnt_off, const int64_t* ex,
                                const int64_t* blk_out, const int64_t* node_off, MemOut mo, int64_t* edge_index,
                                int64_t* edge_type, int64_t* edge_time) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_hits) return;
  const Hit h = hits[i];
  const int64_t mbk = h.x;
  const int m = (int)(mbk / n_blocks), b = (int)(mbk % n_blocks);
  if (blk_out[mbk] < 0) return;
  const int T = blocks[b].tgt_type, S = blocks[b].src_type;
  const auto mb = member(st, m);
  const int64_t r = h.y, sser = h.w;
  const int64_t* noff = node_off + (int64_t)m * st.num_types;
  const int64_t eb = mo.edge_base(m);
  const int64_t o = blk_out[mbk] + ex[cnt_off[mbk] + r] - ex[cnt_off[mbk]] + h.z;
  const int64_t tid = st.lid[mb.lid_off[T] + r], sid = st.lid[mb.lid_off[S] + sser];
  edge_index[mo.src_pos(m) + o] = noff[S] + sser;                        // row 0 = source (data.py:245,254)
  edge_index[mo.dst_pos(m) + o] = noff[T] + r;
  edge_type[eb + o] = blocks[b].rel;
  edge_time[eb + o] = node_ltime(st, mb, T, tid, r) - node_ltime(st, mb, S, sid, sser) + 120;   // data.py:250
}

// k_rb_nodes with the feature rows read from host memory: 16-byte loads when the row and the output row are 16-byte
// aligned (feat_dim % 4 == 0 and aligned tables), kRowUnroll of them per lane issued before the first store.
template <class St>
__global__ void k_rb_nodes_host(St st, const int64_t* node_off, const int64_t* type_out,
                                const int64_t* self_off, int64_t self_rel, MemOut mo, const float* const* feat,
                                int32_t feat_dim, int64_t* node_type, int64_t* node_time, float* node_feature,
                                int64_t* edge_index, int64_t* edge_type, int64_t* edge_time) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int t = blockIdx.y;
  const int m = blockIdx.z;
  const auto mb = member(st, m);
  const int64_t noff = node_off[(int64_t)m * st.num_types + t];
  if (noff < 0 || r >= mb.n_layer[t]) return;
  const int64_t lrow = noff + r;
  const int64_t row = mo.node_base(m) + lrow;
  const int64_t tid = st.lid[mb.lid_off[t] + r];
  if (lane == 0) {
    node_type[row] = type_out[t];
    node_time[row] = node_ltime(st, mb, t, tid, r);
    const int64_t so = self_off[(int64_t)m * st.num_types + t];
    if (so >= 0) {
      const int64_t e = so + r, eb = mo.edge_base(m);
      edge_index[mo.src_pos(m) + e] = lrow;
      edge_index[mo.dst_pos(m) + e] = lrow;
      edge_type[eb + e] = self_rel;
      edge_time[eb + e] = 120;
    }
  }
  if (!node_feature) return;
  const float* src = feat[t] + tid * (int64_t)feat_dim;
  float* dst = node_feature + row * (int64_t)feat_dim;
  if ((feat_dim & 3) == 0 && (((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    const int n4 = feat_dim >> 2;
    for (int c0 = 0; c0 < n4; c0 += 32 * kRowUnroll) {
      float4 v[kRowUnroll];
#pragma unroll
      for (int u = 0; u < kRowUnroll; ++u)
        if (c0 + 32 * u + lane < n4) v[u] = s4[c0 + 32 * u + lane];
#pragma unroll
      for (int u = 0; u < kRowUnroll; ++u)
        if (c0 + 32 * u + lane < n4) d4[c0 + 32 * u + lane] = v[u];
    }
  } else {
    for (int c0 = 0; c0 < feat_dim; c0 += 32 * kRowUnroll) {
      float v[kRowUnroll];
#pragma unroll
      for (int u = 0; u < kRowUnroll; ++u)
        if (c0 + 32 * u + lane < feat_dim) v[u] = src[c0 + 32 * u + lane];
#pragma unroll
      for (int u = 0; u < kRowUnroll; ++u)
        if (c0 + 32 * u + lane < feat_dim) dst[c0 + 32 * u + lane] = v[u];
    }
  }
}

// ---- bf16 feature tables (sampler.py: DeviceGraph(..., feature_dtype=torch.bfloat16)) --------------------------------
// The widening is exact: a bf16 value is the high half of the float's bits.
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// One warp per output row i: node_feature[i] = widen(feat[row_type[i]][row_id[i]]).  Elements before the row's first
// 16-byte boundary and after its last are copied one by one; between them each lane keeps kRowUnroll 16-byte loads (8
// values each) in flight, so a table in host memory is read in whole 16-byte requests at any width.
__global__ void k_gather_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                              const int64_t* row_id, int64_t n_rows, float* node_feature) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (i >= n_rows || row_id[i] < 0) return;
  const uint16_t* src = feat[row_type[i]] + row_id[i] * (int64_t)feat_dim;
  float* dst = node_feature + i * (int64_t)feat_dim;
  int head = (int)((((uintptr_t)0 - (uintptr_t)src) & 15) >> 1);
  if (head > feat_dim) head = feat_dim;
  const int n8 = (feat_dim - head) >> 3;
  for (int c = lane; c < head; c += 32) dst[c] = bf16_lo(src[c]);
  const uint4* s8 = reinterpret_cast<const uint4*>(src + head);
  float* d8 = dst + head;
  const bool vec_store = ((uintptr_t)d8 & 15) == 0;
  for (int c0 = 0; c0 < n8; c0 += 32 * kRowUnroll) {
    uint4 v[kRowUnroll];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u)
      if (c0 + 32 * u + lane < n8) v[u] = s8[c0 + 32 * u + lane];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int c = c0 + 32 * u + lane;
      if (c >= n8) continue;
      const float4 a = make_float4(bf16_lo(v[u].x), bf16_hi(v[u].x), bf16_lo(v[u].y), bf16_hi(v[u].y));
      const float4 b = make_float4(bf16_lo(v[u].z), bf16_hi(v[u].z), bf16_lo(v[u].w), bf16_hi(v[u].w));
      float* d = d8 + 8 * (int64_t)c;
      if (vec_store) {
        reinterpret_cast<float4*>(d)[0] = a;
        reinterpret_cast<float4*>(d)[1] = b;
      } else {
        d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w;
        d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
      }
    }
  }
  for (int c = head + 8 * n8 + lane; c < feat_dim; c += 32) dst[c] = bf16_lo(src[c]);
}

// One warp per output row i: node_feature[i] = feat[row_type[i]][row_id[i]] as stored, bf16 (sampler.py:
// sample_subgraph(s)_cuda(..., feature_dtype=torch.bfloat16)).  Loads as k_gather_bf16's: 16 bytes at a time from the
// row's first 16-byte boundary on.  A store takes 16 bytes where the destination is 16-byte aligned at that point, 4
// where it is 4-byte aligned, 2 otherwise (source and destination rows may sit at different phases when the width is
// not a multiple of 8).
__global__ void k_gather_rows_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                                   const int64_t* row_id, int64_t n_rows, uint16_t* node_feature) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (i >= n_rows || row_id[i] < 0) return;
  const uint16_t* src = feat[row_type[i]] + row_id[i] * (int64_t)feat_dim;
  uint16_t* dst = node_feature + i * (int64_t)feat_dim;
  int head = (int)((((uintptr_t)0 - (uintptr_t)src) & 15) >> 1);
  if (head > feat_dim) head = feat_dim;
  const int n8 = (feat_dim - head) >> 3;
  for (int c = lane; c < head; c += 32) dst[c] = src[c];
  const uint4* s8 = reinterpret_cast<const uint4*>(src + head);
  uint16_t* d8 = dst + head;
  const int phase = (uintptr_t)d8 & 15;
  for (int c0 = 0; c0 < n8; c0 += 32 * kRowUnroll) {
    uint4 v[kRowUnroll];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u)
      if (c0 + 32 * u + lane < n8) v[u] = s8[c0 + 32 * u + lane];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int c = c0 + 32 * u + lane;
      if (c >= n8) continue;
      uint16_t* d = d8 + 8 * (int64_t)c;
      if (phase == 0) {
        *reinterpret_cast<uint4*>(d) = v[u];
      } else if ((phase & 3) == 0) {
        uint32_t* d4 = reinterpret_cast<uint32_t*>(d);
        d4[0] = v[u].x; d4[1] = v[u].y; d4[2] = v[u].z; d4[3] = v[u].w;
      } else {
        const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) d[2 * j] = (uint16_t)w[j], d[2 * j + 1] = (uint16_t)(w[j] >> 16);
      }
    }
  }
  for (int c = head + 8 * n8 + lane; c < feat_dim; c += 32) dst[c] = src[c];
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
  int32_t *vals_in, *vals_out, *mkey_in, *mkey_out;
  unsigned long long* count;
  uint64_t *okey_in, *okey_out;                                         // hashed: (member, id) order of the entries
  int64_t *oent_in, *oent_out;
  void* cub_tmp;
  size_t cub_bytes;
};

// One member sorts its n ids with one radix sort; B > 1 members add a stable sort by member (mkey) after it.  The hashed
// selection sorts its n region entries by (member, id) first.
size_t carve_select(SelectScratch& s, void* base, int64_t n, int32_t n_members, bool hashed = false) {
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
  s.mkey_in = s.mkey_out = nullptr;
  if (n_members > 1) {
    s.mkey_in = (int32_t*)take(sizeof(int32_t) * (n + 1));
    s.mkey_out = (int32_t*)take(sizeof(int32_t) * (n + 1));
  }
  s.count = (unsigned long long*)take(sizeof(unsigned long long) * n_members);
  s.okey_in = s.okey_out = nullptr;
  s.oent_in = s.oent_out = nullptr;
  if (hashed) {
    s.okey_in = (uint64_t*)take(sizeof(uint64_t) * (n + 1));
    s.okey_out = (uint64_t*)take(sizeof(uint64_t) * (n + 1));
    s.oent_in = (int64_t*)take(sizeof(int64_t) * (n + 1));
    s.oent_out = (int64_t*)take(sizeof(int64_t) * (n + 1));
  }
  s.cub_bytes = 0;
  cub::DeviceRadixSort::SortPairsDescending(nullptr, s.cub_bytes, (const double*)nullptr, (double*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1));
  if (n_members > 1) {
    size_t b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b2, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr,
                                    (int32_t*)nullptr, (int)(n + 1));
    s.cub_bytes = s.cub_bytes > b2 ? s.cub_bytes : b2;
  }
  if (hashed) {
    size_t b3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b3, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int64_t*)nullptr,
                                    (int64_t*)nullptr, (int)(n + 1));
    s.cub_bytes = s.cub_bytes > b3 ? s.cub_bytes : b3;
  }
  s.cub_tmp = take(s.cub_bytes);
  return off;
}

inline int64_t blocks_for(int64_t n, int per = kThreads) { return (n + per - 1) / per; }

int budget_bytes(int32_t n_members, int64_t max_targets, int32_t n_blocks, int64_t sampled_number, size_t* out_bytes,
                 const char* what) {
  HGT_REQUIRE(out_bytes && n_members >= 1 && n_members < 65536 && max_targets >= 0 && n_blocks >= 0 &&
                  sampled_number > 0,
              "%s: bad arguments", what);
  const int64_t n_seg = max_targets * n_blocks * n_members;
  HGT_REQUIRE(n_seg < (int64_t(1) << 31) && n_seg * sampled_number < (int64_t(1) << 40),
              "%s: %d members x %lld targets x %d blocks x width %lld is too large", what, n_members,
              (long long)max_targets, n_blocks, (long long)sampled_number);
  BudgetScratch s;
  *out_bytes = carve_budget(s, nullptr, n_seg, n_seg * sampled_number);
  return 0;
}

template <class St>
int add_budget(const St& hs, const int64_t* step, const hgt_gsample_block* blocks, BlockRange br, int32_t max_blocks,
               const int64_t* tgt_id, const int64_t* tgt_time, int64_t max_targets, const int64_t* n_targets,
               int64_t sampled_number, int32_t time_filter, int64_t max_time, int64_t no_time, int32_t* flags,
               void* workspace, size_t workspace_bytes, void* stream, const char* what) {
  const int64_t S = max_targets * max_blocks;
  if (S == 0) return 0;
  size_t need = 0;
  if (int rc = budget_bytes(hs.n_members, max_targets, max_blocks, sampled_number, &need, what)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n_seg = S * hs.n_members;
  const int64_t cap = n_seg * sampled_number;
  BudgetScratch s;
  carve_budget(s, workspace, n_seg, cap);
  k_seg_count<<<blocks_for(n_seg + 1), kThreads, 0, st>>>(blocks, br, hs.n_members, S, tgt_id, max_targets, n_targets,
                                                         sampled_number, s.seg_cnt);
  HGT_LAUNCH_CHECK();
  size_t tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(s.cub_tmp, tmp, s.seg_cnt, s.seg_off, (int)(n_seg + 1), st));
  k_candidates<<<blocks_for(n_seg, kWarps), kThreads, 0, st>>>(
      hs, step, blocks, br, S, tgt_id, tgt_time, max_targets, s.seg_cnt, s.seg_off, sampled_number, time_filter,
      max_time, no_time, s.cand_pos, s.cand_slot, s.cand_time, flags);
  HGT_LAUNCH_CHECK();
  const int64_t gx = blocks_for(cap / hs.n_members);
  const int64_t gx_max = 1024 / hs.n_members > 4 ? 1024 / hs.n_members : 4;
  k_resolve<<<dim3((unsigned)(gx < gx_max ? gx : gx_max), hs.n_members), kThreads, 0, st>>>(hs, step, s.seg_off, S,
                                                                                           s.cand_slot, s.cand_time);
  HGT_LAUNCH_CHECK();
  k_touch<<<(unsigned)blocks_for(hs.n_members, 32), 32, 0, st>>>(hs);
  HGT_LAUNCH_CHECK();
  return 0;
}

int select_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes, const char* what) {
  HGT_REQUIRE(out_bytes && n_members >= 1 && n_members < 65536 && n_total >= 0 && n_total < (int64_t(1) << 31) - 1,
              "%s: %lld ids of %d members do not fit int32 sort values", what, (long long)n_total, n_members);
  SelectScratch s;
  *out_bytes = carve_select(s, nullptr, n_total, n_members);
  return 0;
}

inline int bits_for(int n) {
  int bits = 0;
  while ((1 << bits) < n) ++bits;
  return bits;
}

// The keys_in / vals_in pairs of a selection sorted by key, descending and stable, then (B > 1) stably by member: each
// member's positions end up together in key order, at the member's sel_off.
int sort_keys(SelectScratch& s, int64_t n_total, int B, const int64_t* sel_off, cudaStream_t st,
              const int32_t** vals) {
  size_t tmp = s.cub_bytes;
  HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairsDescending(s.cub_tmp, tmp, s.keys_in, s.keys_out, s.vals_in,
                                                           s.vals_out, (int)n_total, 0, 64, st));
  *vals = s.vals_out;
  if (B > 1) {
    k_sel_member<<<blocks_for(n_total), kThreads, 0, st>>>(sel_off, B, s.vals_out, n_total, s.mkey_in);
    HGT_LAUNCH_CHECK();
    tmp = s.cub_bytes;
    HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, s.mkey_in, s.mkey_out, s.vals_out, s.vals_in,
                                                   (int)n_total, 0, bits_for(B), st));
    *vals = s.vals_in;
  }
  return 0;
}

int select(const hgt_gsample_batch_state& hs, const int32_t* type, const int64_t* step, const int64_t* sel_off,
           int64_t n_total, int64_t max_ids, int64_t sampled_number, int64_t* tgt_id, int64_t* tgt_time,
           int64_t* n_targets, int32_t* flags, void* workspace, size_t workspace_bytes, void* stream,
           const char* what) {
  size_t need = 0;
  if (int rc = select_bytes(hs.n_members, n_total, &need, what)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, need);
  const int B = hs.n_members;
  cudaStream_t st = (cudaStream_t)stream;
  SelectScratch s;
  carve_select(s, workspace, n_total, B);
  HGT_CHECK_CUDA(cudaMemsetAsync(s.count, 0, sizeof(unsigned long long) * B, st));
  if (n_total > 0 && max_ids > 0) {
    const int64_t g = blocks_for(max_ids);
    k_sel_count<<<dim3((unsigned)(g < 1024 ? g : 1024), B), kThreads, 0, st>>>(hs, type, s.count);
    HGT_LAUNCH_CHECK();
    k_sel_keys<<<dim3((unsigned)g, B), kThreads, 0, st>>>(hs, type, sel_off, sampled_number, s.count, step, s.keys_in,
                                                          s.vals_in);
    HGT_LAUNCH_CHECK();
    const int32_t* vals = nullptr;
    if (int rc = sort_keys(s, n_total, B, sel_off, st, &vals)) return rc;
    k_sel_take<<<dim3((unsigned)blocks_for(sampled_number), B), kThreads, 0, st>>>(
        hs, type, sel_off, sampled_number, s.count, vals, tgt_id, tgt_time, flags);
    HGT_LAUNCH_CHECK();
  }
  k_sel_finish<<<(unsigned)blocks_for(B, 32), 32, 0, st>>>(hs, type, sampled_number, s.count, n_targets);
  HGT_LAUNCH_CHECK();
  return 0;
}

int hash_select_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes, const char* what) {
  HGT_REQUIRE(out_bytes && n_members >= 1 && n_members < 65536 && n_total >= 0 && n_total < (int64_t(1) << 31) - 1,
              "%s: %lld entries of %d members do not fit int32 sort values", what, (long long)n_total, n_members);
  SelectScratch s;
  *out_bytes = carve_select(s, nullptr, n_total, n_members, true);
  return 0;
}

int hash_select(const hgt_gsample_hash_state& hs, const int32_t* type, const int64_t* step, const int64_t* sel_off,
                int64_t n_total, int64_t max_room, int64_t sampled_number, int64_t* tgt_id, int64_t* tgt_time,
                int64_t* n_targets, int32_t* flags, void* workspace, size_t workspace_bytes, void* stream,
                const char* what) {
  size_t need = 0;
  if (int rc = hash_select_bytes(hs.n_members, n_total, &need, what)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, need);
  const int B = hs.n_members;
  cudaStream_t st = (cudaStream_t)stream;
  SelectScratch s;
  carve_select(s, workspace, n_total, B, true);
  HGT_CHECK_CUDA(cudaMemsetAsync(s.count, 0, sizeof(unsigned long long) * B, st));
  if (n_total > 0 && max_room > 0) {
    const int64_t g = blocks_for(max_room);
    k_hsel_order<<<dim3((unsigned)(g < 1024 ? g : 1024), B), kThreads, 0, st>>>(hs, type, sel_off, max_room, n_total,
                                                                                 s.okey_in, s.oent_in, s.count);
    HGT_LAUNCH_CHECK();
    size_t tmp = s.cub_bytes;
    HGT_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(s.cub_tmp, tmp, s.okey_in, s.okey_out, s.oent_in, s.oent_out,
                                                   (int)n_total, 0, kIdBits + bits_for(B), st));
    k_hsel_keys<<<dim3((unsigned)g, B), kThreads, 0, st>>>(hs, type, sel_off, max_room, n_total, sampled_number,
                                                           s.count, step, s.okey_out, s.oent_out, s.keys_in, s.vals_in);
    HGT_LAUNCH_CHECK();
    const int32_t* vals = nullptr;
    if (int rc = sort_keys(s, n_total, B, sel_off, st, &vals)) return rc;
    k_hsel_take<<<dim3((unsigned)blocks_for(sampled_number), B), kThreads, 0, st>>>(
        hs, type, sel_off, sampled_number, s.count, vals, s.oent_out, tgt_id, tgt_time, flags);
    HGT_LAUNCH_CHECK();
  }
  k_sel_finish<<<(unsigned)blocks_for(B, 32), 32, 0, st>>>(hs, type, sampled_number, s.count, n_targets);
  HGT_LAUNCH_CHECK();
  return 0;
}

// n_hits != NULL: the single-read count pass of a host-resident graph, leaving up to hit_cap hit records in `hits`.
template <class St>
int rebuild_count(const St& hs, const hgt_gsample_block* blocks, int32_t n_blocks,
                  const int64_t* min_ser, const int64_t* cnt_off, int64_t n_count, int64_t max_rows,
                  const int64_t* feat_rows, Hit* hits, int64_t hit_cap, unsigned long long* n_hits, int64_t* ex,
                  int64_t* totals, int32_t* flags, void* workspace, size_t workspace_bytes, void* stream,
                  const char* what) {
  HGT_REQUIRE(n_blocks >= 0 && n_blocks < 65536 && hs.num_types < 65536 && hs.n_members >= 1 &&
                  hs.n_members < 65536 && max_rows >= 0,
              "%s: bad arguments", what);
  size_t need = 0;
  if (int rc = hgt_gsample_rebuild_workspace_bytes(n_count, &need)) return rc;
  HGT_REQUIRE(workspace && workspace_bytes >= need, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* cnt = (int64_t*)workspace;
  void* cub_tmp = (char*)workspace + hgt_align_up(sizeof(int64_t) * (n_count + 1), 256);
  size_t tmp = workspace_bytes - hgt_align_up(sizeof(int64_t) * (n_count + 1), 256);
  HGT_CHECK_CUDA(cudaMemsetAsync(cnt + n_count, 0, sizeof(int64_t), st));
  if (n_hits) {
    HGT_CHECK_CUDA(cudaMemsetAsync(n_hits, 0, sizeof(unsigned long long), st));
    if (n_blocks > 0 && max_rows > 0) {
      k_rb_count_host<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_blocks, hs.n_members), kThreads, 0, st>>>(
          hs, blocks, n_blocks, min_ser, cnt_off, cnt, hits, hit_cap, n_hits, flags);
      HGT_LAUNCH_CHECK();
    }
  } else if (n_blocks > 0 && max_rows > 0) {
    k_rb_count<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_blocks, hs.n_members), kThreads, 0, st>>>(
        hs, blocks, n_blocks, min_ser, cnt_off, cnt, flags);
    HGT_LAUNCH_CHECK();
  }
  HGT_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, tmp, cnt, ex, (int)(n_count + 1), st));
  const int64_t n_tot = (int64_t)n_blocks * hs.n_members;
  if (n_tot > 0) {
    k_rb_totals<<<blocks_for(n_tot), kThreads, 0, st>>>(ex, cnt_off, n_tot, totals);
    HGT_LAUNCH_CHECK();
  }
  if (feat_rows && max_rows > 0 && hs.num_types > 0) {
    k_rb_check_features<<<dim3((unsigned)blocks_for(max_rows), hs.num_types, hs.n_members), kThreads, 0, st>>>(
        hs, feat_rows, flags);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

// host_graph: the instances for a host-resident graph (k_rb_write_hits over the n_hits records in `hits`, or k_rb_write
// when hits is NULL; k_rb_nodes_host).
template <class St>
int rebuild_write(const St& hs, const hgt_gsample_block* blocks, int32_t n_blocks,
                  const int64_t* min_ser, const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out,
                  const int64_t* node_off,
                  const int64_t* type_out, const int64_t* self_off, int64_t self_rel, MemOut mo, int64_t max_rows,
                  bool host_graph, const Hit* hits, int64_t n_hits,
                  const float* const* feat, int32_t feat_dim, int64_t* node_type, int64_t* node_time,
                  float* node_feature, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time, void* stream,
                  const char* what) {
  HGT_REQUIRE(n_blocks >= 0 && n_blocks < 65536 && hs.num_types < 65536 && hs.n_members >= 1 &&
                  hs.n_members < 65536 && max_rows >= 0 && feat_dim >= 0 && (node_feature == nullptr || feat != nullptr),
              "%s: bad arguments", what);
  cudaStream_t st = (cudaStream_t)stream;
  if (max_rows == 0) return 0;
  if (hits) {
    if (n_hits > 0) {
      k_rb_write_hits<<<(unsigned)blocks_for(n_hits), kThreads, 0, st>>>(hs, blocks, n_blocks, hits, n_hits, cnt_off, ex,
                                                                        blk_out, node_off, mo, edge_index, edge_type,
                                                                        edge_time);
      HGT_LAUNCH_CHECK();
    }
  } else if (n_blocks > 0) {
    k_rb_write<<<dim3((unsigned)blocks_for(max_rows, kWarps), n_blocks, hs.n_members), kThreads, 0, st>>>(
        hs, blocks, n_blocks, min_ser, cnt_off, ex, blk_out, node_off, mo, edge_index, edge_type, edge_time);
    HGT_LAUNCH_CHECK();
  }
  if (hs.num_types > 0) {
    const dim3 grid((unsigned)blocks_for(max_rows, kWarps), hs.num_types, hs.n_members);
    if (host_graph)
      k_rb_nodes_host<<<grid, kThreads, 0, st>>>(hs, node_off, type_out, self_off, self_rel, mo, feat, feat_dim,
                                                 node_type, node_time, node_feature, edge_index, edge_type, edge_time);
    else
      k_rb_nodes<<<grid, kThreads, 0, st>>>(hs, node_off, type_out, self_off, self_rel, mo, feat, feat_dim, node_type,
                                            node_time, node_feature, edge_index, edge_type, edge_time);
    HGT_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace

// ---- the dense state ------------------------------------------------------------------------------------------------

extern "C" int hgt_gsample_batch_add_budget_workspace_bytes(int32_t n_members, int64_t max_targets, int32_t max_blocks,
                                                            int64_t sampled_number, size_t* out_bytes) {
  return budget_bytes(n_members, max_targets, max_blocks, sampled_number, out_bytes,
                      "hgt_gsample_batch_add_budget_workspace_bytes");
}

extern "C" int hgt_gsample_batch_add_budget(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                            const int32_t* type_blocks, int32_t max_blocks, const int32_t* type,
                                            const int64_t* step, const int64_t* tgt_id, const int64_t* tgt_time,
                                            int64_t max_targets, const int64_t* n_targets, int64_t sampled_number,
                                            int32_t time_filter, int64_t max_time, int64_t no_time, int32_t* flags,
                                            void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && h_state->seed && type_blocks && type && step && n_targets && sampled_number > 0 &&
                  max_targets >= 0 && max_blocks >= 0,
              "hgt_gsample_batch_add_budget: bad arguments");
  return add_budget(*h_state, step, blocks, {type_blocks, type}, max_blocks, tgt_id, tgt_time, max_targets, n_targets,
                    sampled_number, time_filter, max_time, no_time, flags, workspace, workspace_bytes, stream,
                    "hgt_gsample_batch_add_budget");
}

extern "C" int hgt_gsample_batch_select_workspace_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes) {
  return select_bytes(n_members, n_total, out_bytes, "hgt_gsample_batch_select_workspace_bytes");
}

extern "C" int hgt_gsample_batch_select(const hgt_gsample_batch_state* h_state, const int32_t* type,
                                        const int64_t* step, const int64_t* sel_off, int64_t n_total, int64_t max_ids,
                                        int64_t sampled_number, int64_t* tgt_id, int64_t* tgt_time, int64_t* n_targets,
                                        int32_t* flags, void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && h_state->seed && type && step && sel_off && sampled_number > 0 && max_ids >= 0,
              "hgt_gsample_batch_select: bad arguments");
  return select(*h_state, type, step, sel_off, n_total, max_ids, sampled_number, tgt_id, tgt_time, n_targets, flags,
                workspace, workspace_bytes, stream, "hgt_gsample_batch_select");
}

extern "C" int hgt_gsample_rebuild_workspace_bytes(int64_t n_count, size_t* out_bytes) {
  HGT_REQUIRE(out_bytes && n_count >= 0 && n_count < (int64_t(1) << 31) - 1,
              "hgt_gsample_rebuild_workspace_bytes: bad count %lld", (long long)n_count);
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(n_count + 1));
  *out_bytes = hgt_align_up(sizeof(int64_t) * (n_count + 1), 256) + b;
  return 0;
}

extern "C" int hgt_gsample_batch_rebuild_count(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                               int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                               int64_t n_count, int64_t max_rows, const int64_t* feat_rows,
                                               int64_t* ex, int64_t* totals, int32_t* flags, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state, "hgt_gsample_batch_rebuild_count: bad arguments");
  return rebuild_count(*h_state, blocks, n_blocks, min_ser, cnt_off, n_count, max_rows, feat_rows, nullptr, 0, nullptr,
                       ex, totals, flags, workspace, workspace_bytes, stream, "hgt_gsample_batch_rebuild_count");
}

extern "C" int hgt_gsample_batch_rebuild_write(
    const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks, int32_t n_blocks, const int64_t* min_ser,
    const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
    const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows, const float* const* feat,
    int32_t feat_dim, int64_t* node_type, int64_t* node_time, float* node_feature, int64_t* edge_index,
    int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(h_state && mem_out, "hgt_gsample_batch_rebuild_write: bad arguments");
  return rebuild_write(*h_state, blocks, n_blocks, min_ser, cnt_off, ex, blk_out, node_off, type_out, self_off,
                       self_rel, {mem_out}, max_rows, false, nullptr, 0, feat, feat_dim, node_type, node_time,
                       node_feature, edge_index, edge_type, edge_time, stream, "hgt_gsample_batch_rebuild_write");
}

// ---- graphs in page-locked host memory ------------------------------------------------------------------------------

extern "C" int hgt_host_register(void* host, size_t bytes, void** dev_ptr) {
  HGT_REQUIRE(host && bytes > 0 && dev_ptr, "hgt_host_register: bad arguments");
  HGT_CHECK_CUDA(cudaHostRegister(host, bytes, cudaHostRegisterMapped));
  const cudaError_t e = cudaHostGetDevicePointer(dev_ptr, host, 0);
  if (e != cudaSuccess) {
    cudaHostUnregister(host);
    hgt_set_error("hgt_host_register: cudaHostGetDevicePointer failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return 0;
}

extern "C" int hgt_host_unregister(void* host) {
  HGT_REQUIRE(host, "hgt_host_unregister: bad arguments");
  HGT_CHECK_CUDA(cudaHostUnregister(host));
  return 0;
}

extern "C" int hgt_gsample_batch_rebuild_count_host(const hgt_gsample_batch_state* h_state,
                                                    const hgt_gsample_block* blocks, int32_t n_blocks,
                                                    const int64_t* min_ser, const int64_t* cnt_off, int64_t n_count,
                                                    int64_t max_rows, const int64_t* feat_rows, void* hits,
                                                    int64_t hit_cap, int64_t* n_hits, int64_t* ex, int64_t* totals,
                                                    int32_t* flags, void* workspace, size_t workspace_bytes,
                                                    void* stream) {
  HGT_REQUIRE(h_state && n_hits && hit_cap >= 0 && hit_cap < (int64_t(1) << 31) && (hits || hit_cap == 0) &&
                  (int64_t)n_blocks * h_state->n_members < (int64_t(1) << 31),
              "hgt_gsample_batch_rebuild_count_host: bad arguments");
  return rebuild_count(*h_state, blocks, n_blocks, min_ser, cnt_off, n_count, max_rows, feat_rows, (Hit*)hits, hit_cap,
                       (unsigned long long*)n_hits, ex, totals, flags, workspace, workspace_bytes, stream,
                       "hgt_gsample_batch_rebuild_count_host");
}

extern "C" int hgt_gsample_batch_rebuild_write_host(
    const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks, int32_t n_blocks, const int64_t* min_ser,
    const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
    const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows, const void* hits,
    int64_t n_hits, const float* const* feat, int32_t feat_dim, int64_t* node_type, int64_t* node_time,
    float* node_feature, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(h_state && mem_out && n_hits >= 0, "hgt_gsample_batch_rebuild_write_host: bad arguments");
  return rebuild_write(*h_state, blocks, n_blocks, min_ser, cnt_off, ex, blk_out, node_off, type_out, self_off,
                       self_rel, {mem_out}, max_rows, true, (const Hit*)hits, n_hits, feat, feat_dim, node_type,
                       node_time, node_feature, edge_index, edge_type, edge_time, stream,
                       "hgt_gsample_batch_rebuild_write_host");
}

// ---- the hashed state -------------------------------------------------------------------------------------------------

extern "C" int hgt_gsample_hash_insert_seeds(const hgt_gsample_hash_state* h_state, int64_t n, const int64_t* region,
                                             const int64_t* id, const int64_t* ser, const int64_t* time, int32_t* flags,
                                             void* stream) {
  HGT_REQUIRE(h_state && h_state->num_types > 0 && n >= 0 && (n == 0 || (region && id && ser && time && flags)),
              "hgt_gsample_hash_insert_seeds: bad arguments");
  if (n == 0) return 0;
  k_hash_seed<<<(unsigned)blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*h_state, n, region, id, ser, time, flags);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_hash_add_budget(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                           const int32_t* type_blocks, int32_t max_blocks, const int32_t* type,
                                           const int64_t* step, const int64_t* tgt_id, const int64_t* tgt_time,
                                           int64_t max_targets, const int64_t* n_targets, int64_t sampled_number,
                                           int32_t time_filter, int64_t max_time, int64_t no_time, int32_t* flags,
                                           void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && h_state->seed && type_blocks && type && step && n_targets && sampled_number > 0 &&
                  max_targets >= 0 && max_blocks >= 0,
              "hgt_gsample_hash_add_budget: bad arguments");
  return add_budget(*h_state, step, blocks, {type_blocks, type}, max_blocks, tgt_id, tgt_time, max_targets, n_targets,
                    sampled_number, time_filter, max_time, no_time, flags, workspace, workspace_bytes, stream,
                    "hgt_gsample_hash_add_budget");
}

extern "C" int hgt_gsample_hash_select_workspace_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes) {
  return hash_select_bytes(n_members, n_total, out_bytes, "hgt_gsample_hash_select_workspace_bytes");
}

extern "C" int hgt_gsample_hash_select(const hgt_gsample_hash_state* h_state, const int32_t* type, const int64_t* step,
                                       const int64_t* sel_off, int64_t n_total, int64_t max_room,
                                       int64_t sampled_number, int64_t* tgt_id, int64_t* tgt_time, int64_t* n_targets,
                                       int32_t* flags, void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state && h_state->seed && type && step && sel_off && sampled_number > 0 && max_room >= 0 &&
                  n_total <= (int64_t)h_state->n_members * max_room,
              "hgt_gsample_hash_select: bad arguments");
  return hash_select(*h_state, type, step, sel_off, n_total, max_room, sampled_number, tgt_id, tgt_time, n_targets,
                     flags, workspace, workspace_bytes, stream, "hgt_gsample_hash_select");
}

extern "C" int hgt_gsample_hash_rebuild_count(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                              int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                              int64_t n_count, int64_t max_rows, const int64_t* feat_rows, int64_t* ex,
                                              int64_t* totals, int32_t* flags, void* workspace,
                                              size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(h_state, "hgt_gsample_hash_rebuild_count: bad arguments");
  return rebuild_count(*h_state, blocks, n_blocks, min_ser, cnt_off, n_count, max_rows, feat_rows, nullptr, 0, nullptr,
                       ex, totals, flags, workspace, workspace_bytes, stream, "hgt_gsample_hash_rebuild_count");
}

extern "C" int hgt_gsample_hash_rebuild_write(
    const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks, int32_t n_blocks, const int64_t* min_ser,
    const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
    const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows, const float* const* feat,
    int32_t feat_dim, int64_t* node_type, int64_t* node_time, float* node_feature, int64_t* edge_index,
    int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(h_state && mem_out, "hgt_gsample_hash_rebuild_write: bad arguments");
  return rebuild_write(*h_state, blocks, n_blocks, min_ser, cnt_off, ex, blk_out, node_off, type_out, self_off,
                       self_rel, {mem_out}, max_rows, false, nullptr, 0, feat, feat_dim, node_type, node_time,
                       node_feature, edge_index, edge_type, edge_time, stream, "hgt_gsample_hash_rebuild_write");
}

extern "C" int hgt_gsample_hash_rebuild_count_host(const hgt_gsample_hash_state* h_state,
                                                   const hgt_gsample_block* blocks, int32_t n_blocks,
                                                   const int64_t* min_ser, const int64_t* cnt_off, int64_t n_count,
                                                   int64_t max_rows, const int64_t* feat_rows, void* hits,
                                                   int64_t hit_cap, int64_t* n_hits, int64_t* ex, int64_t* totals,
                                                   int32_t* flags, void* workspace, size_t workspace_bytes,
                                                   void* stream) {
  HGT_REQUIRE(h_state && n_hits && hit_cap >= 0 && hit_cap < (int64_t(1) << 31) && (hits || hit_cap == 0) &&
                  (int64_t)n_blocks * h_state->n_members < (int64_t(1) << 31),
              "hgt_gsample_hash_rebuild_count_host: bad arguments");
  return rebuild_count(*h_state, blocks, n_blocks, min_ser, cnt_off, n_count, max_rows, feat_rows, (Hit*)hits, hit_cap,
                       (unsigned long long*)n_hits, ex, totals, flags, workspace, workspace_bytes, stream,
                       "hgt_gsample_hash_rebuild_count_host");
}

extern "C" int hgt_gsample_hash_rebuild_write_host(
    const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks, int32_t n_blocks, const int64_t* min_ser,
    const int64_t* cnt_off, const int64_t* ex, const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
    const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows, const void* hits,
    int64_t n_hits, const float* const* feat, int32_t feat_dim, int64_t* node_type, int64_t* node_time,
    float* node_feature, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time, void* stream) {
  HGT_REQUIRE(h_state && mem_out && n_hits >= 0, "hgt_gsample_hash_rebuild_write_host: bad arguments");
  return rebuild_write(*h_state, blocks, n_blocks, min_ser, cnt_off, ex, blk_out, node_off, type_out, self_off,
                       self_rel, {mem_out}, max_rows, true, (const Hit*)hits, n_hits, feat, feat_dim, node_type,
                       node_time, node_feature, edge_index, edge_type, edge_time, stream,
                       "hgt_gsample_hash_rebuild_write_host");
}

// ---- bf16 feature tables ------------------------------------------------------------------------------------------------

extern "C" int hgt_gsample_gather_features_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                                                const int64_t* row_id, int64_t n_rows, float* node_feature,
                                                void* stream) {
  HGT_REQUIRE(feat_dim >= 0 && n_rows >= 0 &&
                  (n_rows == 0 || feat_dim == 0 || (feat && row_type && row_id && node_feature)),
              "hgt_gsample_gather_features_bf16: bad arguments");
  if (n_rows == 0 || feat_dim == 0) return 0;
  k_gather_bf16<<<(unsigned)blocks_for(n_rows, kWarps), kThreads, 0, (cudaStream_t)stream>>>(feat, feat_dim, row_type,
                                                                                           row_id, n_rows, node_feature);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_gather_rows_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                                            const int64_t* row_id, int64_t n_rows, void* node_feature, void* stream) {
  HGT_REQUIRE(feat_dim >= 0 && n_rows >= 0 &&
                  (n_rows == 0 || feat_dim == 0 || (feat && row_type && row_id && node_feature)),
              "hgt_gsample_gather_rows_bf16: bad arguments");
  if (n_rows == 0 || feat_dim == 0) return 0;
  k_gather_rows_bf16<<<(unsigned)blocks_for(n_rows, kWarps), kThreads, 0, (cudaStream_t)stream>>>(
      feat, feat_dim, row_type, row_id, n_rows, static_cast<uint16_t*>(node_feature));
  HGT_LAUNCH_CHECK();
  return 0;
}

// ---- sampling with fixed shapes (sampler.py: GraphedSampler) --------------------------------------------------------
// The host decisions of sample_subgraphs_cuda made on the device, so that a whole call can be captured in a CUDA graph.

namespace {

// One thread per member: its budget types in first-touch order (the reference's list(budget.keys()), data.py:150) as
// steps k = 0.. of this layer, -1 past its last one; step numbers continue the member's counter, which advances by the
// member's number of budget types.
__global__ void k_layer_order(const int64_t* type_seq, int32_t n_members, int32_t num_types, int64_t* next_step,
                              int32_t* type, int64_t* step) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_members) return;
  const int T = num_types, B = n_members;
  const int64_t* ts = type_seq + (int64_t)m * 2 * T;
  int k = 0;
  for (long long last = -1;; ++k) {                                   // the next budget type after first-touch `last`
    int best = -1;
    long long bv = kNoSeq;
    for (int t = 0; t < T; ++t)
      if (ts[2 * t + 1] > last && ts[2 * t + 1] < bv) { bv = ts[2 * t + 1]; best = t; }
    if (best < 0) break;
    type[(int64_t)k * B + m] = best;
    step[(int64_t)k * B + m] = next_step[m] + k;
    last = bv;
  }
  for (int j = k; j < T; ++j) {
    type[(int64_t)j * B + m] = -1;
    step[(int64_t)j * B + m] = next_step[m] + j;
  }
  next_step[m] += k;
}

// After k_layer_order: sel_off [T, B+1] from the chosen regions (one thread per step).
__global__ void k_layer_offsets(int32_t n_members, int32_t num_types, const int64_t* rooms, const int32_t* type,
                                int64_t* sel_off) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= num_types) return;
  const int B = n_members;
  int64_t o = 0;
  for (int m = 0; m < B; ++m) {
    sel_off[(int64_t)k * (B + 1) + m] = o;
    const int t = type[(int64_t)k * B + m];
    if (t >= 0) o += rooms[(int64_t)m * num_types + t];
  }
  sel_off[(int64_t)k * (B + 1) + B] = o;
}

// The to_torch layout of every member (sampler.py: _member_layout) written into a signature's padded layout, members
// joined type-major as merge_batches joins them: member m's type-t rows start at row0[t] + (type-t nodes of the members
// before it), its edges follow the edges of the members before it, and edge_index is one [2, n_edges] array.  One
// thread: B x (T + n_blocks) steps.  A count past a bound, a pair outside the signature, a sampled type without a
// feature table, or any flag the sampler raised empties every table (-1), so the write pass writes nothing.
__global__ void k_graphed_layout(int32_t n_members, int32_t num_types, int32_t n_blocks, const int64_t* n_layer,
                                 const int64_t* type_seq, const int64_t* totals, const int32_t* grp_off,
                                 const int32_t* grp_blk, const int32_t* blk_pair, const int32_t* self_pair,
                                 const int32_t* has_feat, const int64_t* row0, const int64_t* type_cap,
                                 int64_t n_edges, int32_t* flags, int64_t* node_off, int64_t* blk_out,
                                 int64_t* self_off, int64_t* mem_out, int64_t* n_real_edges) {
  if (blockIdx.x || threadIdx.x) return;
  const int B = n_members, T = num_types, NB = n_blocks;
  int64_t eb = 0;
  for (int m = 0; m < B; ++m) {
    const int64_t* nl = n_layer + (int64_t)m * T;
    const int64_t* ts = type_seq + (int64_t)m * 2 * T;
    for (int t = 0; t < T; ++t) {
      int64_t before = 0;
      for (int q = 0; q < m; ++q) before += n_layer[(int64_t)q * T + t];
      node_off[(int64_t)m * T + t] = row0[t] + before;
      self_off[(int64_t)m * T + t] = -1;
      if (before + nl[t] > type_cap[t] && !flags[4]) flags[4] = t + 1;
      if (nl[t] && !has_feat[t] && !flags[7]) flags[7] = t + 1;
    }
    for (int b = 0; b < NB; ++b) blk_out[(int64_t)m * NB + b] = -1;
    int64_t E = 0;
    for (long long last = -1;;) {                                     // layer_data key order (data.py:181-184)
      int tt = -1;
      long long bv = kNoSeq;
      for (int t = 0; t < T; ++t)
        if (ts[2 * t] > last && ts[2 * t] < bv) { bv = ts[2 * t]; tt = t; }
      if (tt < 0) break;
      last = bv;
      if (nl[tt] == 0) continue;
      self_off[(int64_t)m * T + tt] = E;
      E += nl[tt];
      if (self_pair[tt] > 0 && !flags[6]) flags[6] = self_pair[tt];
      for (int g = grp_off[tt]; g < grp_off[tt + 1]; ++g) {
        const int b = grp_blk[g];
        const int64_t n = totals[(int64_t)m * NB + b];
        if (!n) continue;
        blk_out[(int64_t)m * NB + b] = E;
        E += n;
        if (blk_pair[b] > 0 && !flags[6]) flags[6] = blk_pair[b];
      }
    }
    mem_out[4 * m] = 0;
    mem_out[4 * m + 1] = eb;
    mem_out[4 * m + 2] = eb;
    mem_out[4 * m + 3] = n_edges + eb;
    eb += E;
  }
  if (eb > n_edges) flags[5] = 1;
  bool bad = false;
  for (int f = 0; f < 8; ++f) bad |= flags[f] != 0;
  *n_real_edges = bad ? 0 : eb;
  if (!bad) return;
  for (int64_t i = 0; i < (int64_t)B * T; ++i) node_off[i] = self_off[i] = -1;
  for (int64_t i = 0; i < (int64_t)B * NB; ++i) blk_out[i] = -1;
}

// The sampled id of every laid-out row (node_id, -1 stays on the rest).  One thread per <member (z), type (y), ser>.
template <class St>
__global__ void k_graphed_rows(St st, const int64_t* node_off, int64_t* node_id) {
  const int t = blockIdx.y, m = blockIdx.z;
  const auto mb = member(st, m);
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t noff = node_off[(int64_t)m * st.num_types + t];
  if (noff < 0 || r >= mb.n_layer[t]) return;
  node_id[noff + r] = st.lid[mb.lid_off[t] + r];
}

// Edges from n_real on become self loops on pad_node with type 0 and time 120 (graphed.py: _Graphed._scatter); when a
// flag is set every feature value becomes NaN.
__global__ void k_graphed_pad(const int64_t* n_real, int64_t n_edges, int64_t pad_node, const int32_t* flags,
                              int64_t* edge_index, int64_t* edge_type, int64_t* edge_time, void* feature,
                              int64_t n_values, int32_t bf16) {
  const int64_t e0 = *n_real;
  bool bad = false;
  for (int f = 0; f < 8; ++f) bad |= flags[f] != 0;
  const int64_t n = n_values > n_edges ? n_values : n_edges;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (i >= e0 && i < n_edges) {
      edge_index[i] = pad_node;
      edge_index[n_edges + i] = pad_node;
      edge_type[i] = 0;
      edge_time[i] = 120;
    }
    if (bad && i < n_values) {
      if (bf16)
        reinterpret_cast<uint16_t*>(feature)[i] = 0x7fc0;
      else
        reinterpret_cast<float*>(feature)[i] = __int_as_float(0x7fc00000);
    }
  }
}

}  // namespace

extern "C" int hgt_gsample_layer_order(const int64_t* type_seq, int32_t n_members, int32_t num_types,
                                       const int64_t* rooms, int64_t* next_step, int32_t* type, int64_t* step,
                                       int64_t* sel_off, void* stream) {
  HGT_REQUIRE(type_seq && rooms && next_step && type && step && sel_off && n_members >= 1 && n_members < 65536 &&
                  num_types >= 1 && num_types < 65536,
              "hgt_gsample_layer_order: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  k_layer_order<<<(unsigned)blocks_for(n_members, 32), 32, 0, st>>>(type_seq, n_members, num_types, next_step, type,
                                                                     step);
  HGT_LAUNCH_CHECK();
  k_layer_offsets<<<(unsigned)blocks_for(num_types, 32), 32, 0, st>>>(n_members, num_types, rooms, type, sel_off);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_graphed_layout(int32_t n_members, int32_t num_types, int32_t n_blocks,
                                          const int64_t* n_layer, const int64_t* type_seq, const int64_t* totals,
                                          const int32_t* grp_off, const int32_t* grp_blk, const int32_t* blk_pair,
                                          const int32_t* self_pair, const int32_t* has_feat, const int64_t* row0,
                                          const int64_t* type_cap, int64_t n_edges, int32_t* flags, int64_t* node_off,
                                          int64_t* blk_out, int64_t* self_off, int64_t* mem_out,
                                          int64_t* n_real_edges, void* stream) {
  HGT_REQUIRE(n_members >= 1 && num_types >= 1 && n_blocks >= 0 && n_edges >= 0 && n_layer && type_seq && totals &&
                  grp_off && (grp_blk || n_blocks == 0) && (blk_pair || n_blocks == 0) && self_pair && has_feat &&
                  row0 && type_cap && flags && node_off && (blk_out || n_blocks == 0) && self_off && mem_out &&
                  n_real_edges,
              "hgt_gsample_graphed_layout: bad arguments");
  k_graphed_layout<<<1, 32, 0, (cudaStream_t)stream>>>(n_members, num_types, n_blocks, n_layer, type_seq, totals,
                                                       grp_off, grp_blk, blk_pair, self_pair, has_feat, row0, type_cap,
                                                       n_edges, flags, node_off, blk_out, self_off, mem_out,
                                                       n_real_edges);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_graphed_rows(const hgt_gsample_hash_state* h_state, const int64_t* node_off,
                                        int64_t max_rows, int64_t* node_id, void* stream) {
  HGT_REQUIRE(h_state && node_off && node_id && max_rows >= 0 && h_state->num_types < 65536 &&
                  h_state->n_members >= 1 && h_state->n_members < 65536,
              "hgt_gsample_graphed_rows: bad arguments");
  if (max_rows == 0 || h_state->num_types == 0) return 0;
  k_graphed_rows<<<dim3((unsigned)blocks_for(max_rows), h_state->num_types, h_state->n_members), kThreads, 0,
                   (cudaStream_t)stream>>>(*h_state, node_off, node_id);
  HGT_LAUNCH_CHECK();
  return 0;
}

extern "C" int hgt_gsample_graphed_pad(const int64_t* n_real_edges, int64_t n_edges, int64_t pad_node,
                                       const int32_t* flags, int64_t* edge_index, int64_t* edge_type,
                                       int64_t* edge_time, void* feature, int64_t n_values, int32_t bf16,
                                       void* stream) {
  HGT_REQUIRE(n_real_edges && flags && n_edges >= 0 && n_values >= 0 &&
                  (n_edges == 0 || (edge_index && edge_type && edge_time)) && (n_values == 0 || feature),
              "hgt_gsample_graphed_pad: bad arguments");
  const int64_t n = n_values > n_edges ? n_values : n_edges;
  if (n == 0) return 0;
  const int64_t g = blocks_for(n);
  k_graphed_pad<<<(unsigned)(g < 2048 ? g : 2048), kThreads, 0, (cudaStream_t)stream>>>(
      n_real_edges, n_edges, pad_node, flags, edge_index, edge_type, edge_time, feature, n_values, bf16);
  HGT_LAUNCH_CHECK();
  return 0;
}
