// One C-ABI call for a whole HGTConv forward (inference): gather (if the node types are not pre-sorted) ->
// weight fold -> typed projections (+ RTE tables) -> fused edge kernel -> typed a_linear -> gated skip + LayerNorm.
// The caller hands over the plan arrays, the parameter pointer tables and ONE workspace; everything is enqueued on
// the given stream without any host synchronisation.  This is what a non-Python host binds for the layer
// (reference boundary: HGTConv.forward, pyHGT/conv.py:56-134); the Python class uses it too, so that a layer costs
// one ctypes call instead of a dozen (the reference's sampled-subgraph batches are launch/host-bound).
// linear_impl 3 runs the tensor-core GEMMs with one bf16 product: the edge kernel then writes gelu(agg) as bf16 hi only,
// and a pre-split x needs no lo half.
// The [K'|V'] and RTE tables take the format hgt_gather_table_format picks: bs16 when the 24-bit table would not fit in
// L2 and d_out % 128 == 0 (hgt_typed_linear_bs16, hgt_edge_forward_bs16; 4.25d bytes per row), else 24-bit when d_out % 8
// == 0 (hgt_typed_linear_t24, hgt_edge_forward_t24; 6d bytes), else fp32.  The projection writes Q as fp32 and the
// K'/V' blocks straight into the table.  A forward that keeps nothing for a backward needs no more than that precision
// (DESIGN.md §4.2, §4.3), and the edge pass reads fewer bytes per edge.
#include "common.cuh"

int hgt_update_epilogue_impl(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                             const float* skip, const float* norm_w, const float* norm_b, const float* const* norm_wp,
                             const float* const* norm_bp, const int32_t* perm, const int32_t* type_active,
                             const int32_t* type_dst, const float* bias, int64_t n_nodes, int32_t d, float* out,
                             void* out_hi, void* out_lo, const uint64_t* seed, float p, cudaStream_t st);
bool hgt_typed_linear_tc_supported(int64_t lda, int32_t K, int32_t cb_width);

namespace {

struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* b) : base(reinterpret_cast<char*>(b)) {}
  template <typename T>
  T* take(size_t count) {
    size_t o = off;
    off += hgt_align_up(count * sizeof(T), 256);
    return base ? reinterpret_cast<T*>(base + o) : nullptr;
  }
  void* take_bytes(size_t bytes) { return take<char>(bytes); }
};

struct Layout {
  float *x_sorted, *w_cat, *b_cat, *proj, *rt, *g_act, *wa_cat, *ba_cat, *o;
  void *kv, *kvr;                                          // fp32 (inside proj), 24-bit or bs16 tables
  void *g_hi, *g_lo, *ws_proj, *ws_edge, *ws_upd;
  size_t ws_proj_bytes, ws_edge_bytes, ws_upd_bytes, total;
  size_t row_bytes;                                        // of a [K'|V'] or RTE table row
  int32_t fmt;                                             // HGT_TABLE_*
  bool fuse_split, presplit_x;
};

int plan_layout(const hgt_conv_args* a, void* base, Layout* L) {
  Carver c(base);
  const int64_t N = a->n_nodes;
  const int d = a->d_out, din = a->d_in;
  HGT_REQUIRE(a->linear_impl >= 0 && a->linear_impl <= 3, "hgt_conv_forward: unknown linear_impl %d", a->linear_impl);
  const bool one = a->linear_impl == 3;                    // one bf16 product: no lo halves
  const bool tc_upd = a->linear_impl != 1 && hgt_typed_linear_tc_supported(d, d, d);
  L->fuse_split = tc_upd;                                  // edge kernel writes gelu(agg) as the bf16 hi/lo split
  L->presplit_x = a->x_hi != nullptr && (a->x_lo != nullptr || one) && a->perm == nullptr && a->linear_impl != 1 &&
                  hgt_typed_linear_tc_supported(din, din, d);
  L->x_sorted = a->perm ? c.take<float>((size_t)N * din) : nullptr;
  L->w_cat = c.take<float>((size_t)(a->cat_rows > 0 ? a->cat_rows : 1) * din);
  L->b_cat = c.take<float>((size_t)(a->cat_rows > 0 ? a->cat_rows : 1));
  int dev = 0, l2 = 0;
  HGT_CHECK_CUDA(cudaGetDevice(&dev));
  HGT_CHECK_CUDA(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev));
  int rc = hgt_gather_table_format(d, a->kv_rows + 1, l2, &L->fmt);
  int64_t rbytes = 0;
  if (rc || (rc = hgt_gather_table_row_bytes(L->fmt, 2 * (int64_t)d, &rbytes))) return rc;
  const size_t row_bytes = L->row_bytes = (size_t)rbytes;
  if (L->fmt != HGT_TABLE_F32) {
    L->proj = c.take<float>((size_t)a->kv_off);           // Q only
    L->kv = c.take_bytes((size_t)(a->kv_rows + 1) * row_bytes);
  } else {
    L->proj = c.take<float>((size_t)a->proj_elems);
    L->kv = base ? L->proj + a->kv_off : nullptr;
  }
  if (L->presplit_x)
    rc = hgt_typed_linear_presplit_workspace_bytes(a->h_proj_groups, a->n_proj_groups, din, d, &L->ws_proj_bytes);
  else
    rc = hgt_typed_linear_workspace_bytes(a->h_proj_groups, a->n_proj_groups, din, d, a->linear_impl, &L->ws_proj_bytes);
  if (rc) return rc;
  L->ws_proj = c.take_bytes(L->ws_proj_bytes + 256);
  L->rt = nullptr;
  L->kvr = nullptr;
  if (a->use_rte) {
    L->rt = c.take<float>((size_t)HGT_RTE_MAX_LEN * din);
    L->kvr = c.take_bytes(((size_t)a->n_pairs * HGT_RTE_MAX_LEN + 1) * row_bytes);
  }
  if ((rc = hgt_edge_workspace_bytes(a->n_split, d, a->n_heads, &L->ws_edge_bytes))) return rc;
  L->ws_edge = c.take_bytes(L->ws_edge_bytes);
  L->g_act = nullptr;
  L->g_hi = L->g_lo = nullptr;
  if (L->fuse_split) {
    L->g_hi = c.take_bytes((size_t)N * d * 2);
    L->g_lo = one ? nullptr : c.take_bytes((size_t)N * d * 2);
  } else {
    L->g_act = c.take<float>((size_t)N * d);
  }
  L->wa_cat = c.take<float>((size_t)a->num_types * d * d);
  L->ba_cat = c.take<float>((size_t)a->num_types * d);
  if (L->fuse_split)
    rc = hgt_typed_linear_presplit_workspace_bytes(a->h_upd_groups, a->n_upd_groups, d, d, &L->ws_upd_bytes);
  else
    rc = hgt_typed_linear_workspace_bytes(a->h_upd_groups, a->n_upd_groups, d, d, a->linear_impl, &L->ws_upd_bytes);
  if (rc) return rc;
  L->ws_upd = c.take_bytes(L->ws_upd_bytes + 256);
  L->o = c.take<float>((size_t)N * d);
  L->total = c.off + 256;
  return 0;
}

}  // namespace

extern "C" int hgt_gather_table_format(int32_t d, int64_t table_rows, int64_t l2_bytes, int32_t* out_format) {
  HGT_REQUIRE(out_format, "hgt_gather_table_format: out_format is NULL");
  // d % 128 == 0: the projection's tiles are 128 or 256 columns wide and every one stores its scales as a whole
  // TMA box; the staged epilogue's scattered 8-byte scale stores (d = 400) cost the projection more than the edge
  // pass gains
  if (d % 128 == 0 && table_rows * 6 * (int64_t)d > l2_bytes) *out_format = HGT_TABLE_BS16;
  else *out_format = d % 8 == 0 ? HGT_TABLE_T24 : HGT_TABLE_F32;
  return 0;
}

extern "C" int hgt_gather_table_row_bytes(int32_t format, int64_t n, int64_t* out_bytes) {
  HGT_REQUIRE(out_bytes, "hgt_gather_table_row_bytes: out_bytes is NULL");
  HGT_REQUIRE(format == HGT_TABLE_F32 || format == HGT_TABLE_T24 || format == HGT_TABLE_BS16,
              "hgt_gather_table_row_bytes: unknown format %d", format);
  *out_bytes = format == HGT_TABLE_BS16 ? hgt_bs16_row_bytes(n) : n * (format == HGT_TABLE_T24 ? 3 : 4);
  return 0;
}

extern "C" uint64_t hgt_conv_args_size(void) { return sizeof(hgt_conv_args); }

extern "C" int hgt_conv_workspace_bytes(const hgt_conv_args* a, size_t* out_bytes) {
  HGT_REQUIRE(a && out_bytes, "hgt_conv_workspace_bytes: NULL argument");
  Layout L;
  int rc = plan_layout(a, nullptr, &L);
  if (rc) return rc;
  *out_bytes = L.total;
  return 0;
}

extern "C" int hgt_conv_forward(const hgt_conv_args* a, void* workspace, size_t workspace_bytes, void* stream) {
  HGT_REQUIRE(a && workspace, "hgt_conv_forward: NULL argument");
  HGT_REQUIRE(a->d_in == a->d_out, "hgt_conv_forward: in_dim must equal out_dim (conv.py:131)");
  HGT_REQUIRE(!a->use_rte || a->rte_row, "hgt_conv_forward: use_rte needs rte_row");
  HGT_REQUIRE(!(a->type_active && a->type_dst), "hgt_conv_forward: type_active and type_dst exclude each other");
  cudaStream_t st = (cudaStream_t)stream;
  Layout L;
  void* base = reinterpret_cast<void*>(hgt_align_up(reinterpret_cast<size_t>(workspace), 256));
  int rc = plan_layout(a, base, &L);
  if (rc) return rc;
  HGT_REQUIRE(workspace_bytes >= L.total, "hgt_conv_forward: workspace too small (%zu < %zu)", workspace_bytes, L.total);
  const int64_t N = a->n_nodes;
  const int d = a->d_out, din = a->d_in, T = a->num_types, P = a->n_pairs;
  if (N == 0) return 0;

  const float* x_sorted = a->x;
  if (a->perm) {
    if ((rc = hgt_gather_rows(a->x, a->perm, N, din, L.x_sorted, stream))) return rc;
    x_sorted = L.x_sorted;
  }
  if ((rc = hgt_fold_weights(a->wq, a->bq, a->wk, a->bk, a->wv, a->bv, a->relation_att, a->relation_msg,
                             a->relation_pri, T, a->num_relations, a->n_heads, din, d, P, a->pair_type, a->pair_rel,
                             a->cat_row0, a->q_row0, L.w_cat, L.b_cat, stream)))
    return rc;
  // trailing all-zero [K'|V'] row (edges that match no <s,t,r> triple); zero encodes to zero bytes
  const size_t row_bytes = L.row_bytes;
  HGT_CHECK_CUDA(cudaMemsetAsync(static_cast<char*>(L.kv) + a->kv_rows * row_bytes, 0, row_bytes, st));
  const void* x_lo = a->linear_impl == 3 ? nullptr : a->x_lo;
  if (L.fmt == HGT_TABLE_BS16) {
    // Q blocks (out_off < kv_off) as fp32, the K'/V' blocks straight into the bs16 table
    if (L.presplit_x)
      rc = hgt_typed_linear_presplit_bs16(a->x_hi, x_lo, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups,
                                          a->n_proj_groups, a->proj_cblocks, L.proj, a->kv_off, L.kv, L.ws_proj,
                                          L.ws_proj_bytes + 256, stream);
    else
      rc = hgt_typed_linear_bs16(x_sorted, din, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups,
                                 a->n_proj_groups, a->proj_cblocks, L.proj, a->kv_off, L.kv, a->linear_impl, L.ws_proj,
                                 L.ws_proj_bytes + 256, stream);
  } else if (L.fmt == HGT_TABLE_T24) {
    // Q blocks (out_off < kv_off) as fp32, the K'/V' blocks straight into the 24-bit table
    if (L.presplit_x)
      rc = hgt_typed_linear_presplit_t24(a->x_hi, x_lo, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups,
                                         a->n_proj_groups, a->proj_cblocks, L.proj, a->kv_off, L.kv, L.ws_proj,
                                         L.ws_proj_bytes + 256, stream);
    else
      rc = hgt_typed_linear_t24(x_sorted, din, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups,
                                a->n_proj_groups, a->proj_cblocks, L.proj, a->kv_off, L.kv, a->linear_impl, L.ws_proj,
                                L.ws_proj_bytes + 256, stream);
  } else if (L.presplit_x) {
    rc = hgt_typed_linear_presplit(a->x_hi, x_lo, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups,
                                   a->n_proj_groups, a->proj_cblocks, L.proj, L.ws_proj, L.ws_proj_bytes + 256, stream);
  } else {
    rc = hgt_typed_linear(x_sorted, din, L.w_cat, L.b_cat, din, d, a->proj_groups, a->h_proj_groups, a->n_proj_groups,
                          a->proj_cblocks, L.proj, a->linear_impl, L.ws_proj, L.ws_proj_bytes + 256, stream);
  }
  if (rc) return rc;
  if (a->use_rte) {
    if ((rc = hgt_typed_linear(a->emb_weight, din, a->emb_lin_w, a->emb_lin_b, din, din, a->rt_groups, a->h_rt_groups, 1,
                               a->rt_cblocks, L.rt, 1, nullptr, 0, stream)))
      return rc;
    HGT_CHECK_CUDA(cudaMemsetAsync(static_cast<char*>(L.kvr) + (int64_t)P * HGT_RTE_MAX_LEN * row_bytes, 0, row_bytes, st));
    if (L.fmt == HGT_TABLE_BS16)
      rc = hgt_typed_linear_bs16(L.rt, din, L.w_cat, nullptr, din, d, a->rte_groups, a->h_rte_groups, a->n_rte_groups,
                                 a->rte_cblocks, nullptr, 0, L.kvr, 1, nullptr, 0, stream);
    else if (L.fmt == HGT_TABLE_T24)
      rc = hgt_typed_linear_t24(L.rt, din, L.w_cat, nullptr, din, d, a->rte_groups, a->h_rte_groups, a->n_rte_groups,
                                a->rte_cblocks, nullptr, 0, L.kvr, 1, nullptr, 0, stream);
    else
      rc = hgt_typed_linear(L.rt, din, L.w_cat, nullptr, din, d, a->rte_groups, a->h_rte_groups, a->n_rte_groups,
                            a->rte_cblocks, static_cast<float*>(L.kvr), 1, nullptr, 0, stream);
    if (rc) return rc;
  }
  // rows past type_dst[t] have no in-edges: as type_active, the edge kernel skips them (their Q rows were not computed)
  const int32_t* dst_rows = a->type_active ? a->type_active : a->type_dst;
  const int32_t* rte_row = a->use_rte ? a->rte_row : nullptr;
  if (L.fmt == HGT_TABLE_BS16)
    rc = hgt_edge_forward_bs16(L.proj + a->q_off, L.kv, L.kvr, a->row_ptr, a->kv_row, rte_row, a->csr_eid, a->tiles,
                               a->n_tiles, a->n_split, a->hubs, a->n_hubs, N, a->n_edges, d, a->n_heads, 1, L.g_act,
                               a->att, nullptr, L.g_hi, L.g_lo, L.ws_edge, L.ws_edge_bytes, a->edge_variant,
                               a->d_tile_counts, a->type_row0, T, dst_rows, stream);
  else if (L.fmt == HGT_TABLE_T24)
    rc = hgt_edge_forward_t24(L.proj + a->q_off, L.kv, L.kvr, a->row_ptr, a->kv_row, rte_row, a->csr_eid, a->tiles,
                              a->n_tiles, a->n_split, a->hubs, a->n_hubs, N, a->n_edges, d, a->n_heads, 1, L.g_act,
                              a->att, nullptr, L.g_hi, L.g_lo, L.ws_edge, L.ws_edge_bytes, a->edge_variant,
                              a->d_tile_counts, a->type_row0, T, dst_rows, stream);
  else
    rc = hgt_edge_forward(L.proj + a->q_off, static_cast<const float*>(L.kv), static_cast<const float*>(L.kvr),
                          a->row_ptr, a->kv_row, rte_row, a->csr_eid, a->tiles, a->n_tiles, a->n_split, a->hubs,
                          a->n_hubs, N, a->n_edges, d, a->n_heads, 1, L.g_act, a->att, nullptr, L.g_hi, L.g_lo,
                          L.ws_edge, L.ws_edge_bytes, a->edge_variant, a->d_tile_counts, a->type_row0, T, dst_rows,
                          stream);
  if (rc) return rc;
  if ((rc = hgt_concat_linears(a->wa, a->ba, T, d, d, L.wa_cat, L.ba_cat, stream))) return rc;
  if (L.fuse_split)
    rc = hgt_typed_linear_presplit(L.g_hi, L.g_lo, L.wa_cat, L.ba_cat, d, d, a->upd_groups, a->h_upd_groups,
                                   a->n_upd_groups, a->upd_cblocks, L.o, L.ws_upd, L.ws_upd_bytes + 256, stream);
  else
    rc = hgt_typed_linear(L.g_act, d, L.wa_cat, L.ba_cat, d, d, a->upd_groups, a->h_upd_groups, a->n_upd_groups,
                          a->upd_cblocks, L.o, a->linear_impl, L.ws_upd, L.ws_upd_bytes + 256, stream);
  if (rc) return rc;
  const int32_t* perm_out = a->out_map ? a->out_map : a->perm;
  return hgt_update_epilogue_impl(L.o, x_sorted, a->type_row0, T, a->skip, nullptr, nullptr,
                                  a->use_norm ? a->norm_w : nullptr, a->use_norm ? a->norm_b : nullptr, perm_out,
                                  a->type_active, a->type_dst, a->type_dst ? L.ba_cat : nullptr, N, d, a->out, a->out_hi,
                                  a->out_lo, nullptr, 0.f, st);
}
