// Host-side helper of pyhgt_b200/sampler.py (HGSampling, reference pyHGT/data.py:87-210).  Plain C++ (no device code):
// the budget update of ONE adjacency slice — data.py:123-130, the loop over the sampled neighbours of one
// <target type, source type, relation> block — done in one call instead of a dozen small numpy operations.
// The random draws stay in numpy (same global RNG stream as the reference); this function is deterministic.
#include "common.cuh"

// ids / tms: the sampled neighbours and their edge times (no_time marks the reference's `None`), in sampling order.
// in_layer [n]: membership of layer_data[source_type];  in_budget / score / b_time / stamp [n]: budget[source_type] as
// flat arrays (stamp reproduces the dict's insertion order);  *stamp_counter: next insertion stamp (shared by all types).
// *touched_layer is set when some candidate passes the time test (the reference then evaluates
// `source_id in layer_data[source_type]`, which creates that defaultdict entry).
// Returns the number of candidates added / updated, or -1 when an id is outside [0, n).
extern "C" int64_t hgt_sampler_budget_update(const int64_t* ids, const int64_t* tms, int64_t n_s, int64_t target_time,
                                             int64_t no_time, int64_t max_time, int64_t n, const uint8_t* in_layer,
                                             uint8_t* in_budget, double* score, int64_t* b_time, int64_t* stamp,
                                             int64_t* stamp_counter, int32_t* touched_layer) {
  for (int64_t i = 0; i < n_s; ++i)                         // validate before touching anything: -1 leaves the state intact
    if (ids[i] < 0 || ids[i] >= n) return -1;
  int64_t kept = 0;
  const double w = 1.0 / (double)n_s;                       // 1. / len(sampled_ids), data.py:129
  for (int64_t i = 0; i < n_s; ++i) {
    const int64_t tm = tms[i] == no_time ? target_time : tms[i];
    if (tm > max_time) continue;                            // data.py:127, first operand of the `or`
    *touched_layer = 1;
    const int64_t id = ids[i];
    if (in_layer[id]) continue;                             // second operand
    if (!in_budget[id]) {                                   // defaultdict creates [0., 0] at the end of the dict
      in_budget[id] = 1;
      score[id] = 0.0;
      stamp[id] = (*stamp_counter)++;
    }
    score[id] += w;
    b_time[id] = tm;
    ++kept;
  }
  return kept;
}

namespace {
// A block's arrays at either width: int64, or int32 with INT32_MIN for no_time (skip & HGT_BLOCK_NARROW).
struct Arrays {
  const hgt_sampler_block& b;
  bool narrow() const { return b.skip & HGT_BLOCK_NARROW; }
  int64_t get(const int64_t* a, int64_t i) const { return narrow() ? (int64_t)((const int32_t*)a)[i] : a[i]; }
  int64_t row_of(int64_t tid) const { return get(b.row_of, tid); }
  int64_t ptr(int64_t row) const { return get(b.ptr, row); }
  int64_t nbr(int64_t j) const { return get(b.nbr, j); }
  int64_t time(int64_t j, int64_t no_time) const {
    if (!narrow()) return b.time[j];
    const int32_t t = ((const int32_t*)b.time)[j];
    return t == INT32_MIN ? no_time : (int64_t)t;
  }
};
}  // namespace

// The whole `add_budget` (data.py:108-130) for a BATCH of target nodes of one type: every <source type, relation> block of
// the target type, in the reference's dict order, target after target — one call per sampling layer and type instead of
// one Python iteration per target and block.  The uniform draws (`np.random.choice(..., replace=False)`, data.py:122) do
// not depend on the budget, so the caller makes them beforehand in the same target-major order and passes the positions
// (draw_off[target * n_blocks + block] = offset into draw_pos, -1 when the adjacency is shorter than sampled_number).
// counters: [0] next budget insertion stamp, [1] next first-touch number of layer_data[type], [2] of budget[type] — the
// two orders the reference gets from its defaultdicts.  Every newly inserted id is also appended to the type's `log`
// (ids in stamp order), so `list(budget[type].keys())` is the log filtered by in_budget: no sort.
// Returns 0, -2 for a neighbour id outside the state arrays, -3 for a missing draw.
extern "C" int64_t hgt_sampler_add_budget(const int64_t* target_ids, const int64_t* target_times, int64_t n_targets,
                                          const hgt_sampler_block* blocks, int32_t n_blocks, hgt_sampler_state* states,
                                          int32_t n_states, int64_t sampled_number, const int64_t* draw_off,
                                          const int64_t* draw_pos, int64_t no_time, int64_t max_time, int64_t* counters) {
  for (int64_t t = 0; t < n_targets; ++t) {
    const int64_t tid = target_ids[t], target_time = target_times[t];
    for (int32_t b = 0; b < n_blocks; ++b) {
      const hgt_sampler_block& blk = blocks[b];
      if ((blk.skip & HGT_BLOCK_SKIP) || tid < 0 || tid >= blk.n_row_of) continue;   // 'self', or target_id not in it
      const Arrays ar{blk};
      const int64_t row = ar.row_of(tid);
      if (row < 0) continue;
      const int64_t a = ar.ptr(row), n_adl = ar.ptr(row + 1) - a;
      if (n_adl == 0) continue;
      if (blk.src_state < 0 || blk.src_state >= n_states) return -2;
      hgt_sampler_state& st = states[blk.src_state];
      const bool all = n_adl < sampled_number;                              // data.py:119-122
      const int64_t n_s = all ? n_adl : sampled_number;
      const int64_t off = all ? 0 : (draw_off ? draw_off[t * n_blocks + b] : -1);
      if (off < 0) return -3;
      const double w = 1.0 / (double)n_s;                                   // 1. / len(sampled_ids), data.py:129
      for (int64_t i = 0; i < n_s; ++i) {
        const int64_t j = a + (all ? i : draw_pos[off + i]);
        const int64_t tj = ar.time(j, no_time);
        const int64_t tm = tj == no_time ? target_time : tj;
        if (tm > max_time) continue;                                        // data.py:127, first operand of the `or`
        if (st.layer_seq < 0) st.layer_seq = counters[1]++;                 // layer_data[source_type] springs into being
        const int64_t sid = ar.nbr(j);
        if (sid < 0 || sid >= st.n) return -2;
        if (st.in_layer[sid]) continue;                                     // second operand
        if (st.budget_seq < 0) st.budget_seq = counters[2]++;
        if (!st.in_budget[sid]) {
          st.in_budget[sid] = 1;
          st.score[sid] = 0.0;
          st.stamp[sid] = counters[0]++;
          st.log[st.log_len++] = sid;
        }
        st.score[sid] += w;
        st.b_time[sid] = tm;
      }
    }
  }
  return 0;
}
