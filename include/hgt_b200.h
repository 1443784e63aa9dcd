/* hgt_b200.h — C ABI of libhgt_b200.so: the H100 (sm_90a) implementation of pyHGT's HGTConv
 * message-passing hot path.
 *
 * Boundary being replaced (reference = acbull/pyHGT, paths relative to the reference root):
 *   pyHGT/conv.py:56-58    HGTConv.forward -> MessagePassing.propagate
 *   pyHGT/conv.py:60-111   HGTConv.message  (typed Q/K/V projections, relation_att / relation_msg,
 *                                           relation_pri, torch_geometric.utils.softmax by target)
 *   pyHGT/conv.py:114-134  HGTConv.update   (gelu, typed a_linear, sigmoid(skip) gate, LayerNorm)
 *   pyHGT/conv.py:283-299  RelTemporalEncoding
 *   third-party: torch_geometric 1.3.2 propagate/softmax, torch_scatter 1.3.2 scatter_add/max
 * The reference has no FFI of its own (pure Python); the Python class pyhgt_b200.HGTConv binds these
 * entry points with ctypes (see INTEGRATION.md for the stub a pyHGT maintainer would add).
 *
 * Conventions
 *   - Every function returns 0 on success, non-zero on error; hgt_last_error() then returns a
 *     thread-local, NUL-terminated description.  Nothing throws across the boundary.
 *   - All pointers are DEVICE pointers unless the parameter name starts with `h_`.
 *   - The caller owns every buffer (inputs, outputs, workspaces).  The library never allocates or frees
 *     device memory and never synchronises the stream unless the function's comment says so.
 *   - `stream` is a cudaStream_t passed as void* (so the header needs no CUDA include).
 *   - Internal node order ("rank order"): nodes sorted stably by node type.  rank[n] is the position of
 *     original node n, perm[k] the original id at position k.  All tables (Q, KV, agg) are in rank order.
 */
#ifndef HGT_B200_H
#define HGT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HGT_RTE_MAX_LEN 240 /* RelTemporalEncoding max_len, conv.py:287 */

const char* hgt_last_error(void);
int hgt_abi_version(void);
/* Number of CUDA kernels this library has launched so far in this process (diagnostics / bench.py). */
uint64_t hgt_kernel_launches(void);

/* ------------------------------------------------------------------------------------------------
 * Graph ingest: int64 COO (the tensors pyHGT/data.py:251-256 `to_torch` emits) -> plan arrays.
 * Replaces PyG propagate's per-layer index_select gathers and the T*T*R boolean triple masks
 * (conv.py:71-84) with one destination-sorted CSR built once per graph.
 * ---------------------------------------------------------------------------------------------- */

/* Bytes of scratch needed by hgt_plan_nodes / hgt_plan_edges_sort / hgt_plan_tiles. */
int hgt_plan_workspace_bytes(int64_t n_nodes, int64_t n_edges, size_t* out_bytes);

/* Stable sort of nodes by type.  rank/perm: [N] int32.  type_count: [T+1] int32 (bucket T collects nodes
 * whose type is outside [0,T): the reference leaves their output rows zero, conv.py:120-124).
 * sorted_flag[0] = 1 if node_type was already non-decreasing (then rank = perm = identity). */
int hgt_plan_nodes(const int64_t* node_type, int64_t n_nodes, int32_t num_types,
                   int32_t* rank, int32_t* perm, int32_t* type_count, int32_t* sorted_flag,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Sort edges by destination rank (stable in original edge order).
 *   edge_index [2,E] int64 row-major (row 0 = source j, row 1 = target i; data.py:245,254)
 *   row_ptr [N+1] int32, csr_eid [E] int32 (CSR position -> original edge id),
 *   presence [T*R] int32: 1 where some valid edge has <source_type, relation> (the "pairs"),
 *   flags [4] int32: flags[0] != 0 => an endpoint id was outside [0,N). */
int hgt_plan_edges_sort(const int64_t* edge_index, const int64_t* edge_type, const int64_t* node_type,
                        const int32_t* rank, int64_t n_nodes, int64_t n_edges,
                        int32_t num_types, int32_t num_relations,
                        int32_t* row_ptr, int32_t* csr_eid, int32_t* presence, int32_t* flags,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Destination extent of every node type, from the CSR of hgt_plan_edges_sort: dst_end [T] int32 (zeroed here) =
 * 1 + the rank of the last row of type t that has an in-edge, or 0 if none has.  Every edge counts, also one that
 * matches no <source type, relation> pair.  perm [N]: from hgt_plan_nodes.  Rows of type t at ranks >= dst_end[t] have
 * no in-edges: their aggregate is 0 and the layer output is exact without computing their Q, edge or a_linear rows
 * (hgt_conv_args.type_dst, hgt_update_epilogue_dst).  Nothing is read back or synchronised. */
int hgt_plan_dst_end(const int32_t* row_ptr, const int32_t* perm, const int64_t* node_type, int64_t n_nodes,
                     int32_t num_types, int32_t* dst_end, void* stream);

/* Per-CSR-edge gather indices.
 *   pair_of [T*R] int32: pair id of <source_type, relation> or -1;  pair_row0 [P] int32: first KV-table
 *   row of each pair;  type_row0 [T+1] int32: first rank of each type;  zero_row: index of the all-zero
 *   KV row used for edges that match no triple (score 0, message 0: conv.py:68-69).
 *   kv_row [E] int32;  rte_row [E] int32 (pair*240 + dt, or zero_rte_row) — pass NULL when edge_time is
 *   NULL.  flags[1] != 0 => an edge_time was outside [0,240) (nn.Embedding would raise, conv.py:299). */
int hgt_plan_edges_fill(const int64_t* edge_index, const int64_t* edge_type, const int64_t* edge_time,
                        const int64_t* node_type, const int32_t* rank, const int32_t* csr_eid,
                        int64_t n_nodes, int64_t n_edges, int32_t num_types, int32_t num_relations,
                        const int32_t* pair_of, const int32_t* pair_row0, const int32_t* type_row0,
                        int32_t zero_row, int32_t zero_rte_row,
                        int32_t* kv_row, int32_t* rte_row, int32_t* flags, void* stream);

/* Balanced work tiles for the edge kernel: consecutive destination ranks are grouped until a tile holds
 * about `target_edges` edges; a destination with more than `split_edges` in-edges is cut into several
 * tiles whose partial (max, sum, acc) are merged afterwards.
 *   tiles [max_tiles,4] int32 = {dst_begin, dst_end, edge_begin, edge_end}; for a split destination
 *   the second field is -(partial_slot+1) < 0 and [edge_begin, edge_end) is a sub-range of its segment.
 *   hubs [max_hubs,4] int32 = {dst, first partial slot, pieces, 0} for every split destination;
 *   n_tiles [3] int32 = {number of tiles, number of split (partial) tiles, number of hubs}.
 * Synchronises the stream (returns the counts to the host through h_n_tiles[3]) — unless h_n_tiles is NULL: then
 * nothing is read back or synchronised, the counts stay in d_n_tiles (pass it to the edge kernels as d_tile_counts)
 * and the caller sizes with the bounds  max_tiles >= (2E+N)/(2*target_edges) + 3*(E/split_edges) + 16,
 * max_hubs >= E/split_edges + 1,  split pieces <= 2*(E/split_edges) + 1. */
int hgt_plan_tiles(const int32_t* row_ptr, int64_t n_nodes, int64_t n_edges,
                   int32_t target_edges, int32_t split_edges,
                   int32_t* tiles, int64_t max_tiles, int32_t* hubs, int64_t max_hubs,
                   int32_t* d_n_tiles, int32_t* h_n_tiles,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Source-major index for the deterministic edge backward: the CSR positions [0, n_edges) stably sorted by key[c]
 * (kv_row: rows of the [K'|V'] table, or rte_row: rows of the RTE table), so every owned row lists its edges in CSR order.
 *   src_ptr [n_rows+1]: entries of row r are [src_ptr[r], src_ptr[r+1]); entries whose key is n_rows (the trailing
 *            all-zero row that collects edges matching no triple) lie past src_ptr[n_rows] and get no work;
 *   src_dst [n_edges]: destination (rank order) of every entry;  src_oth [n_edges]: other[c] of every entry, or NULL
 *            together with other.
 * No host read-back; work tiles over it come from hgt_plan_tiles(src_ptr, n_rows, ...) in its sync-free mode.
 * workspace: hgt_plan_workspace_bytes(n_rows, n_edges). */
int hgt_plan_source_index(const int32_t* key, const int32_t* other, const int32_t* row_ptr, int64_t n_nodes,
                          int64_t n_edges, int32_t n_rows, int32_t* src_ptr, int32_t* src_dst, int32_t* src_oth,
                          void* workspace, size_t workspace_bytes, void* stream);
/* The same index, and src_pos [E]: the CSR position of every entry, in index order, from the same sort (the row pass of
 * the att gradient, hgt_edge_backward_rows_att, reads datt there). */
int hgt_plan_source_index_pos(const int32_t* key, const int32_t* other, const int32_t* row_ptr, int64_t n_nodes,
                              int64_t n_edges, int32_t n_rows, int32_t* src_ptr, int32_t* src_dst, int32_t* src_oth,
                              int32_t* src_pos, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Trimmed forward (GNN.forward(..., out_nodes=)): layer l of L only needs the nodes within L-l hops of an output node.
 * ---------------------------------------------------------------------------------------------- */

/* Hop layout of a batch.  dist[v] [N] int32 = min(L+1, length of the shortest directed path (source -> destination)
 * from v to any out_nodes entry), by L edge-parallel passes from the out_nodes.  hop_perm [N] int32: the nodes stably
 * sorted by (type, dist) — types 0..T-1 in order, nodes of a type outside [0,T) last in their original order;
 * hop_rank [N] int32 its inverse; hop_node_type [N] int64 = node_type[hop_perm]; hop_edge_index [2,E] int64 = hop_rank of
 * every endpoint (edge order kept); out_rows [n_out] int64 = hop_rank[out_nodes].
 * meta (int32, zeroed here) = [counts T*(L+2) | presence T*R | flags 4]:
 *   counts[t*(L+2)+b]: nodes of type t with dist == b (b = L+1: farther or unreachable);
 *   presence[s*R+r] = 1 where a valid edge has <source type s, relation r> (as hgt_plan_edges_sort);
 *   flags[0]: an edge endpoint outside [0,N); flags[1]: an edge_time of such an edge outside [0,240) (edge_time may be
 *   NULL); flags[2]: an out_nodes entry outside [0,N) (the outputs derived from it are then meaningless).
 * Nothing is read back or synchronised.  workspace: hgt_plan_workspace_bytes(n_nodes, n_edges). */
int hgt_trim_layout(const int64_t* edge_index, const int64_t* edge_type, const int64_t* edge_time,
                    const int64_t* node_type, int64_t n_nodes, int64_t n_edges, int32_t num_types,
                    int32_t num_relations, const int64_t* out_nodes, int64_t n_out, int32_t n_layers,
                    int32_t* dist, int32_t* hop_perm, int32_t* hop_rank, int64_t* hop_node_type,
                    int64_t* hop_edge_index, int64_t* out_rows, int32_t* meta, void* workspace,
                    size_t workspace_bytes, void* stream);

/* hgt_trim_layout with host-given slot sizes, so that every size derived from the layout is known on the host before
 * the call and nothing needs reading back (a CUDA graph can capture it).  hop_bounds: host int32 [T, L+2].  The n_rows
 * hop rows are, per type in type order, one region of hop_bounds[t][b] rows for every hop class b = 0..L+1, then a tail
 * [sum of the bounds, n_rows) for the nodes of types outside [0,T).  The nodes of a class fill its region in
 * hgt_trim_layout's order; unused rows are padding: hop_perm = n_nodes (gather from a zero row appended to
 * node_feature), hop_node_type = the region's type (T in the tail), no edges.  A node that does not fit its region is
 * dropped (hop_rank = -1): its edge endpoints and out_rows entries become the pad row n_rows-1, and no region is
 * written past its end.  Dropping is harmless for hop class L+1 and the tail (no layer computes those rows or reads
 * them as typed sources) when a tail row exists to serve as the pad; any other drop sets flags[3] (overflow).
 * hop_perm, hop_node_type: [n_rows]; dist, hop_rank: [n_nodes]; hop_edge_index, out_rows as hgt_trim_layout.
 * meta (int32) = [counts T*(L+2) | presence T*R | flags 4 | offsets T*(L+2)+2]: counts, presence and flags[0..2] as
 * hgt_trim_layout (counts are the actual class sizes, whatever the bounds); offsets[k] the first row of region k,
 * offsets[T*(L+2)] the tail's, offsets[T*(L+2)+1] = n_rows.  The bounds reach the device in kernel parameters, not by a
 * host-memory copy.  With bounds equal to the counts and n_rows = n_nodes the outputs are hgt_trim_layout's, bitwise.
 * n_rows >= the sum of the bounds, and >= 1 if n_nodes > 0.  workspace: hgt_plan_workspace_bytes(n_nodes, n_edges). */
int hgt_trim_layout_bounded(const int64_t* edge_index, const int64_t* edge_type, const int64_t* edge_time,
                            const int64_t* node_type, int64_t n_nodes, int64_t n_edges, int32_t num_types,
                            int32_t num_relations, const int64_t* out_nodes, int64_t n_out, int32_t n_layers,
                            const int32_t* hop_bounds, int64_t n_rows, int32_t* dist, int32_t* hop_perm,
                            int32_t* hop_rank, int64_t* hop_node_type, int64_t* hop_edge_index, int64_t* out_rows,
                            int32_t* meta, void* workspace, size_t workspace_bytes, void* stream);

/* hgt_plan_tiles (sync-free mode, same tile / hub / count formats) over the destinations of n_ranges ascending, disjoint
 * row ranges ranges[2j] .. ranges[2j+1] (device int32 [n_ranges,2]) of row_ptr; n_range_rows = total rows in the ranges
 * (host).  No tile crosses a range end, so an edge kernel launched with these tiles reads and writes only the rows of
 * the ranges.  Bounds: max_tiles >= (2E+N)/(2*target_edges) + 3*(E/split_edges) + 16 + n_ranges, max_hubs and split
 * pieces as for hgt_plan_tiles.  workspace: hgt_plan_workspace_bytes(n_nodes, n_edges). */
int hgt_plan_range_tiles(const int32_t* row_ptr, int64_t n_nodes, int64_t n_edges, const int32_t* ranges,
                         int32_t n_ranges, int64_t n_range_rows, int32_t target_edges, int32_t split_edges,
                         int32_t* tiles, int64_t max_tiles, int32_t* hubs, int64_t max_hubs, int32_t* d_n_tiles,
                         void* workspace, size_t workspace_bytes, void* stream);

/* out_key[c] = key[c] for CSR positions c whose destination lies in one of the row ranges (as hgt_plan_range_tiles),
 * no_work_row otherwise: with no_work_row = n_rows, hgt_plan_source_index(out_key, ...) then indexes only the edges of
 * those destinations. */
int hgt_plan_mask_rows(const int32_t* key, const int32_t* row_ptr, const int32_t* ranges, int32_t n_ranges,
                       int64_t n_edges, int32_t no_work_row, int32_t* out_key, void* stream);

/* out[k,:] = in[perm[k],:]  (rows of `width` floats); used only when node_type is not pre-sorted. */
int hgt_gather_rows(const float* in, const int32_t* perm, int64_t n_rows, int32_t width,
                    float* out, void* stream);

/* Multi-GPU halo exchange fused into one kernel: out[i,:] = peer[src_rank[i]][src_row[i],:], where
 * peer_ptrs_dev is the DEVICE address of an array of world_size device pointers to every rank's [rows,width]
 * feature buffer (NVLink peer mappings, e.g. torch symmetric memory `buffer_ptrs_dev`); `row_base` is added to every
 * src_row (double-buffered publish areas inside one symmetric allocation).  The caller orders the ranks: publish ->
 * barrier -> pull; with two publish areas used alternately that ONE barrier per exchange also guarantees that nobody
 * still reads the area about to be overwritten.  Any width: rows of a multiple of 4 floats into a 16-byte aligned `out`
 * move as float4 (the peer buffers are then assumed 16-byte aligned, as allocations are), other rows float by float. */
int hgt_halo_pull(uint64_t peer_ptrs_dev, const int32_t* src_rank, const int32_t* src_row, int64_t n_rows,
                  int32_t width, int64_t row_base, float* out, void* stream);
/* Same pull fused with the operand conversion of the projection GEMM: every row is written as the bf16 hi/lo split
 * (hi/lo [n_rows, width], the A operand of hgt_typed_linear_presplit) while it crosses NVLink; the fp32 copy is kept
 * only for rows owned by `self_rank` (the update epilogue's skip connection reads those).  width % 8 == 0.
 * `order` (NULL = 0..n_rows-1): the sequence in which the rows are processed; a sequence that cycles through the owners
 * (and starts at a different owner on every rank) keeps every NVLink source evenly loaded. */
int hgt_halo_pull_split(uint64_t peer_ptrs_dev, const int32_t* src_rank, const int32_t* src_row,
                        const int32_t* order, int64_t n_rows, int32_t width, int32_t self_rank, int64_t row_base,
                        float* out_f32, void* hi, void* lo, void* stream);

/* Push variant of the fused exchange (experimental): the OWNER converts its rows and stores the bf16 hi/lo split straight
 * into the consumers' operand buffers (posted NVLink writes).  Item i: row push_src[i] of x_own [rows, width] -> row
 * row_base + push_dst[i] of rank push_peer[i]'s hi / lo buffers (hi_ptrs_dev / lo_ptrs_dev: DEVICE arrays of world_size
 * device pointers, peer mappings); items addressed to self_rank also write the fp32 row into x_local_f32.  The caller
 * orders the ranks (push -> barrier -> consume; two destination areas used alternately).  width % 8 == 0. */
int hgt_halo_push_split(const float* x_own, const int32_t* push_peer, const int32_t* push_src, const int32_t* push_dst,
                        int64_t n_items, int32_t width, int32_t self_rank, int64_t row_base, uint64_t hi_ptrs_dev,
                        uint64_t lo_ptrs_dev, float* x_local_f32, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Typed (per-node-type) linear layers — "per-type linear dispatch" (conv.py:73-77,96-97,103,125).
 * ---------------------------------------------------------------------------------------------- */

typedef struct {
  int64_t a_row0;    /* first row of A used by this group                                   */
  int64_t m;         /* rows in this group (nodes of this type; 240 for the RTE tables)      */
  int32_t w_row0;    /* first row of the concatenated weight matrix W [sum n_out, K]         */
  int32_t n_cblocks; /* output column blocks of width `cb_width` each                        */
  int32_t cb_first;  /* index of this group's first entry in the column-block table          */
  int32_t has_bias;
} hgt_lin_group;

typedef struct {
  int64_t out_off;   /* element offset of (group row 0, column 0 of this block) from `out`   */
  int64_t ld;        /* elements between consecutive rows of this block's destination        */
} hgt_lin_cblock;

/* Fold the relation matrices into per-<source type, relation> weights (SURVEY.md §8 a4):
 *   W_cat rows for type t: [ W_q^t ; for each pair p=(t,r): K'_p ; V'_p ]  with
 *   K'_p[h*dk+c,:] = pri[r,h]/sqrt(dk) * sum_a att[r,h,a,c] * W_k^t[h*dk+a,:]   (conv.py:97-99)
 *   V'_p[h*dk+c,:] =                     sum_a msg[r,h,a,c] * W_v^t[h*dk+a,:]   (conv.py:103-104)
 * and the same for the biases.  wq/wk/wv/bq/bk/bv are DEVICE arrays of T device pointers (one
 * nn.Linear per type, conv.py:34-38).  pair_type/pair_rel: [P] int32; cat_row0: [P] int32 first W_cat
 * row of the pair's K' block (V' follows at +d_out); q_row0: [T] int32 first W_cat row of W_q^t. */
int hgt_fold_weights(const float* const* wq, const float* const* bq,
                     const float* const* wk, const float* const* bk,
                     const float* const* wv, const float* const* bv,
                     const float* relation_att, const float* relation_msg, const float* relation_pri,
                     int32_t num_types, int32_t num_relations, int32_t n_heads, int32_t d_in, int32_t d_out,
                     int32_t n_pairs, const int32_t* pair_type, const int32_t* pair_rel,
                     const int32_t* cat_row0, const int32_t* q_row0,
                     float* w_cat, float* b_cat, void* stream);

/* Concatenate T per-type [rows,cols] matrices (and [rows] biases) into one: w_cat [T*rows, cols]. */
int hgt_concat_linears(const float* const* w, const float* const* b, int32_t num_types,
                       int32_t rows, int32_t cols, float* w_cat, float* b_cat, void* stream);

/* RelTemporalEncoding (conv.py:299) needs no entry point of its own: RT = emb.weight @ lin.weight^T + lin.bias
 * [240,d] is one hgt_typed_linear call, and its projection through every pair's K'/V' weights another. */

/* out[cblock c of group g][m, n] = sum_k A[a_row0_g + m, k] * W[w_row0_g + c*cb_width + n, k] (+ bias).
 * fp32 in / fp32 out.  `impl`: 0 = auto, 1 = SIMT fp32 FMA kernel, 2 = wgmma split-bf16 tensor-core
 * kernel (three bf16 products of a hi/lo operand split accumulated in one fp32 register accumulator: accurate
 * to ~1e-5 relative; needs cb_width % 16 == 0 and K >= 64, workspace for the split operands), 3 = auto with ONE bf16
 * product on the tensor cores (both operands rounded to bf16 to nearest-even, products accumulated in fp32: torch's
 * "medium" float32 matmul precision; only the hi halves are made, so the workspace is at most impl 2's) and the fp32
 * SIMT kernel where auto would pick it.  Any other impl is rejected, by the workspace query too.
 * groups/cblocks are DEVICE arrays; h_groups is the same table on the host (used to size the grid; no
 * device read-back). */
int hgt_typed_linear_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K,
                                     int32_t cb_width, int32_t impl, size_t* out_bytes);
int hgt_typed_linear(const float* A, int64_t lda, const float* W, const float* bias, int32_t K,
                     int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                     int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int32_t impl,
                     void* workspace, size_t workspace_bytes, void* stream);
/* Same product on the tensor-core kernel with the A operand already split by its producer: a_hi / a_lo are bf16
 * [rows, K] (K % 8 == 0, row stride K).  Saves the split pass over A (workspace: W split only).  a_lo == NULL selects
 * one bf16 product (a_hi * bf16(W), as impl 3); the workspace query's answer covers both. */
int hgt_typed_linear_presplit_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, int32_t K,
                                              int32_t cb_width, size_t* out_bytes);
int hgt_typed_linear_presplit(const void* a_hi, const void* a_lo, const float* W, const float* bias, int32_t K,
                              int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                              int32_t n_groups, const hgt_lin_cblock* cblocks, float* out,
                              void* workspace, size_t workspace_bytes, void* stream);
/* The same two products with a bf16 output: `out` is bf16 and the column blocks' out_off / ld count bf16 elements.  Same
 * tiles, k order and bias add as the fp32 call; each fp32 result is rounded to nearest-even once when it is stored, so
 * the output equals the fp32 call's output converted to bf16, bitwise.  Workspaces: the fp32 calls' queries. */
int hgt_typed_linear_bf16(const float* A, int64_t lda, const float* W, const float* bias, int32_t K,
                          int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                          int32_t n_groups, const hgt_lin_cblock* cblocks, void* out, int32_t impl,
                          void* workspace, size_t workspace_bytes, void* stream);
int hgt_typed_linear_presplit_bf16(const void* a_hi, const void* a_lo, const float* W, const float* bias, int32_t K,
                                   int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                   int32_t n_groups, const hgt_lin_cblock* cblocks, void* out,
                                   void* workspace, size_t workspace_bytes, void* stream);
/* hgt_typed_linear with a bf16 A (`A` bf16 [rows, K] at row stride lda elements; fp32 output): the same product as the
 * fp32 call on A widened to float, bitwise, with the same impl values.  A bf16 value is exactly the hi half of the split
 * and its lo half is zero, so the tensor cores run A*W_hi + A*W_lo (impl 0 / 2; A*W_hi at impl 3) with A read as the
 * wgmma operand as it is: by TMA in place where K % 8 == 0, lda % 8 == 0 and A is 16-byte aligned, otherwise after a
 * copy into zero-padded rows (stream-ordered memory of its own).  impl 1 (and shapes the tensor cores do not take) runs
 * the SIMT kernel, which widens A as it loads it.  Workspace: hgt_typed_linear_workspace_bytes for the same arguments. */
int hgt_typed_linear_bf16a(const void* A, int64_t lda, const float* W, const float* bias, int32_t K, int32_t cb_width,
                           const hgt_lin_group* groups, const hgt_lin_group* h_groups, int32_t n_groups,
                           const hgt_lin_cblock* cblocks, float* out, int32_t impl, void* workspace,
                           size_t workspace_bytes, void* stream);

/* 24-bit gather tables (inference [K'|V'] and RTE tables).
 * Element: the fp32 bit pattern b rounded to nearest-even at bit 8 (b + 0x7F + ((b >> 8) & 1), low 8 bits cleared):
 * sign, 8-bit exponent and 15 stored mantissa bits, relative error <= 2^-16.  A NaN stays a quiet NaN with its sign,
 * Inf stays Inf, finite values that round past FLT_MAX become Inf; +-0 and subnormals follow the same rule.
 * Storage: the rounded word's bits 31..16 are the element's 16-bit "hi", bits 15..8 its 8-bit "lo"; it decodes to the
 * fp32 word (hi << 16) | (lo << 8).
 * Rows (planar): a table row of n logical elements is [hi x n (u16) | lo x n (u8)], 3n bytes; element c of the row has
 * its hi at byte 2c and its lo at byte 2n + c.  A [K'|V'] row (n = 2d) takes 6d bytes.
 * hgt_typed_linear_t24 / hgt_typed_linear_presplit_t24: the fp32 calls' product (same tiles, k order and bias add).
 * Column blocks with out_off < t24_off are fp32 at out + out_off, as in the fp32 calls (out may be NULL when there are
 * none); the others are 24-bit at out24, each result rounded once into this format as it is stored, so the output equals
 * the fp32 call's output encoded, bitwise.  One call thus writes the Q blocks (fp32) and the K'/V' blocks (24-bit) of
 * the projection table, whose K'/V' blocks start at kv_off.  The 24-bit blocks' out_off - t24_off and ld count logical
 * elements: a block's rows have ld elements each (row stride 3 ld bytes), and out_off - t24_off = row * ld + col places
 * element (row, col) of the table at hi byte row * 3 ld + 2 col and lo byte row * 3 ld + 2 ld + col of out24.
 * Workspaces: the fp32 calls' queries. */
int hgt_typed_linear_t24(const float* A, int64_t lda, const float* W, const float* bias, int32_t K,
                         int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                         int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int64_t t24_off, void* out24,
                         int32_t impl, void* workspace, size_t workspace_bytes, void* stream);
int hgt_typed_linear_presplit_t24(const void* a_hi, const void* a_lo, const float* W, const float* bias, int32_t K,
                                  int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                  int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int64_t t24_off,
                                  void* out24, void* workspace, size_t workspace_bytes, void* stream);

/* bs16 gather tables (inference [K'|V'] and RTE tables that do not fit in L2; see hgt_gather_table_format).
 * Blocks: a row of n logical elements (n % 16 == 0) is cut into blocks of 16 consecutive elements.  For a block with
 * largest |x| = a (fp32):
 *   s = fp32(a * fp32(1/32767)) rounded up to bf16;  r = 1 / s in IEEE fp32, times fp32(1 - 2^-15) when s >= 2^112;
 *   m = rint_even(fp32(x * r)) as int16, |m| <= 32767.
 * The element decodes to m * s, which is exact in fp32 (a 15-bit integer times an 8-bit significand, never past
 * FLT_MAX: that is what the 1 - 2^-15 near the top of the range is for), so a decoded table holds ordinary fp32 values.
 * Special blocks: one whose s would be below FLT_MIN (a < ~3.9e-34, all-zero blocks included) stores s = 0 and m = 0:
 * zero encodes to zero bytes.  One holding a NaN or an Inf stores s = NaN (bf16 0x7FC0) and m = 0, so all its elements
 * decode to NaN: a row that is non-finite in fp32 stays non-finite, a finite row stays finite.
 * Rows (planar): [m x n (int16) | s x n/16 (bf16)], zero-padded to a multiple of 16 bytes: element c has its mantissa
 * at byte 2c and its block's scale at byte 2n + 2 (c / 16).  A [K'|V'] row (n = 2d) takes (4.25 d rounded up to 16) bytes:
 * 1088 at d = 256, 1712 at d = 400, 544 at d = 128.
 * hgt_typed_linear_bs16 / hgt_typed_linear_presplit_bs16: as the _t24 calls (fp32 column blocks before t24_off at out,
 * the others in the table at out16, 16-byte aligned, each block encoded once as it is stored, so the output equals the
 * fp32 call's output encoded, bitwise); a block's rows of ld elements lie hgt_gather_table_row_bytes(HGT_TABLE_BS16, ld)
 * bytes apart.
 * Needs cb_width % 16 == 0, so that no 16-element block straddles two column blocks. */
int hgt_typed_linear_bs16(const float* A, int64_t lda, const float* W, const float* bias, int32_t K,
                          int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                          int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int64_t t24_off, void* out16,
                          int32_t impl, void* workspace, size_t workspace_bytes, void* stream);
int hgt_typed_linear_presplit_bs16(const void* a_hi, const void* a_lo, const float* W, const float* bias, int32_t K,
                                   int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                   int32_t n_groups, const hgt_lin_cblock* cblocks, float* out, int64_t t24_off,
                                   void* out16, void* workspace, size_t workspace_bytes, void* stream);

/* Storage format of an inference forward's [K'|V'] and RTE gather tables (one forward that keeps nothing for a
 * backward, outside bf16 autocast), decided here for both hgt_conv_forward and the per-stage Python path so that they
 * compute the same bits.  table_rows: rows of the [K'|V'] table (trailing zero row included); l2_bytes: the device's
 * L2 size.  *out_format = HGT_TABLE_BS16 where d % 128 == 0 and the 24-bit table would be larger than L2 (the edge pass
 * then reads its rows from HBM, and fewer bytes per row are time saved; at d % 128 == 0 the projection's tensor-store
 * epilogue writes each tile's scales as one TMA box, elsewhere its scattered scale stores cost more than the edge pass
 * gains), HGT_TABLE_T24 where d % 8 == 0 otherwise (an L2-resident table gains nothing from fewer bytes and keeps the
 * smaller error), else HGT_TABLE_F32. */
#define HGT_TABLE_F32 0
#define HGT_TABLE_T24 1
#define HGT_TABLE_BS16 2
int hgt_gather_table_format(int32_t d, int64_t table_rows, int64_t l2_bytes, int32_t* out_format);
/* *out_bytes = the bytes of a table row of n elements in a format: 4n, 3n or the bs16 row */
int hgt_gather_table_row_bytes(int32_t format, int64_t n, int64_t* out_bytes);

/* ------------------------------------------------------------------------------------------------
 * Fused edge kernel: gather -> relation-specific score -> softmax by destination -> weighted sum
 * (conv.py:99,108-111 + PyG scatter-add), one pass over the destination-sorted CSR.
 * ---------------------------------------------------------------------------------------------- */

/*  q       [N, d]        rank order, Q[i] = W_q^{type(i)} x_i + b
 *  kv      [rows+1, 2d]  row = [K' | V'] of <source node, relation>; last row all zero
 *  kvr     [P*240+1, 2d] RTE contribution per <pair, dt> (NULL when !use_RTE); last row all zero
 *  tiles / hubs from hgt_plan_tiles;  partial workspace: n_split slots of round4(2*H) + round4(d) floats
 *          (round4: rounded up to a multiple of 4, which keeps every slot's accumulator 16-byte aligned)
 *  agg_out [N, d]  gelu(sum_e att[e] * V'[e]) if apply_gelu else the raw sum   (conv.py:119)
 *  att_out [E, H]  softmax weights in ORIGINAL edge order (conv.py:108 `self.att`) or NULL
 *  stats_out [N, 2H] per-destination (max, sum) per head, or NULL (kept for the backward pass)
 *  g_hi / g_lo [N, d] bf16 or NULL: the same result as a bf16 hi/lo split (x = hi + lo to ~2^-17), i.e. the
 *           pre-split A operand of hgt_typed_linear_presplit; agg_out may then be NULL.  Needs d % 8 == 0.  g_hi without
 *           g_lo writes the hi half only (the operand of a one-product GEMM, a_lo == NULL).
 *  variant: 0 = auto, 1 = direct register gather (LDG), 2 = bulk-async-copy shared-memory ring (TMA)
 *  d_tile_counts: NULL, or the device counts {n_tiles, n_split, n_hubs} hgt_plan_tiles wrote in its sync-free mode; then
 *           n_tiles / n_split_tiles / n_hubs are the UPPER BOUNDS the arrays were sized with and the kernels read the
 *           true counts from the device (no host read-back between plan build and layer).
 *  type_row0 [T+2] / type_active [T]: NULL, or (sharded runs) the same tables hgt_update_epilogue takes: destinations
 *           past the active prefix of their type are halo sources — they have no in-edges and no output row is written.
 *           The type extents of hgt_plan_dst_end serve as type_active too: the rows past them have no in-edges. */
int hgt_edge_workspace_bytes(int32_t n_split_tiles, int32_t d, int32_t n_heads, size_t* out_bytes);
int hgt_edge_forward(const float* q, const float* kv, const float* kvr,
                     const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                     const int32_t* csr_eid, const int32_t* tiles, int32_t n_tiles, int32_t n_split_tiles,
                     const int32_t* hubs, int32_t n_hubs,
                     int64_t n_nodes, int64_t n_edges, int32_t d, int32_t n_heads, int32_t apply_gelu,
                     float* agg_out, float* att_out, float* stats_out, void* g_hi, void* g_lo,
                     void* workspace, size_t workspace_bytes, int32_t variant, const int32_t* d_tile_counts,
                     const int32_t* type_row0, int32_t num_types, const int32_t* type_active, void* stream);

/* Backward of hgt_edge_forward (training; the reference differentiates the same ops with autograd,
 * OAG/train_paper_field.py:249).  Inputs: the forward's q / kv / kvr tables, its un-activated output
 * `agg` (apply_gelu = 0), the saved per-destination softmax statistics `stats` [N,2H] and the incoming
 * gradient `dagg` [N,d].  Outputs (ZERO-INITIALISED BY THIS CALL, on the stream): dq [N,d],
 * dkv [kv_rows_total, 2d] (gradient of the [K'|V'] table; kv_rows_total counts the trailing all-zero row, whose
 * gradient is to be discarded), dkvr [kvr_rows_total, 2d] or NULL.  workspace: >= 256 bytes. */
int hgt_edge_backward(const float* q, const float* kv, const float* kvr, const float* agg, const float* dagg,
                      const float* stats, const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                      const int32_t* tiles, int32_t n_tiles, int64_t n_nodes, int32_t d, int32_t n_heads,
                      int64_t kv_rows_total, int64_t kvr_rows_total,
                      float* dq, float* dkv, float* dkvr, void* workspace, size_t workspace_bytes,
                      const int32_t* d_tile_counts, void* stream);

/* Deterministic backward of hgt_edge_forward: the same gradients without float atomics, bitwise repeatable.
 * hgt_edge_backward_dst: destination pass.  Writes dq [N,d] (zero-initialised here; hub pieces go to partial rows in the
 *   workspace and are summed in piece order through `hubs`) and D [N,H] = <dagg_i, agg_i> per head (rows of
 *   destinations without in-edges are not written).  Does not touch the K'/V' gradients.
 * hgt_edge_backward_rows: row pass over a source-major index (hgt_plan_source_index + hgt_plan_tiles).  One warp owns a
 *   row of `own` ([own_rows_total, 2d]: the [K'|V'] table keyed by kv_row, or the RTE table keyed by rte_row) and walks its
 *   entries in order: it gathers Q_i, dagg_i, (m, l)_i, D_i and the row src_oth[j] of `oth` (the other table, added to
 *   the key / value row as in the forward; NULL without RTE), and writes grad[row] = [sum ds Q_i | sum p dagg_i] with
 *   one store.  Rows [n_rows, own_rows_total) (the trailing all-zero row) are zeroed.  Split rows: partial rows summed
 *   in piece order.
 *   In place: grad may be `own` itself (fp32 tables, hgt_edge_backward_rows[_att]; the bf16 entry points have an fp32
 *   grad and a bf16 own, which never alias).  The result is then bitwise that of a separate grad.  This holds because
 *   every read of own[r] precedes every write of grad[r]: the owning warp loads its row before walking the row's
 *   entries and stores it once at the end; the pieces of a split row (every piece of it is split) read the row and write
 *   workspace partials, which a later launch sums into grad[r]; a row without entries loads nothing and stores zeros;
 *   rows past n_rows are zeroed before the pass and never read as `own`; own is read with coherent loads.  `oth` must
 *   not alias grad: the RTE row pass reads the [K'|V'] rows as oth, so it runs before an in-place [K'|V'] pass.
 * tiles / n_tiles / n_split / hubs / n_hubs / d_tile_counts as for hgt_edge_forward (for the row pass: from
 *   hgt_plan_tiles over src_ptr).  Every d / n_heads that hgt_edge_backward takes is supported.
 * workspace: hgt_edge_backward_det_workspace_bytes(n_split of the destination tiles, n_split of the row tiles, d); the
 *   passes run one after the other on the stream, so one workspace serves all of them. */
int hgt_edge_backward_det_workspace_bytes(int32_t n_split_dst, int32_t n_split_rows, int32_t d, size_t* out_bytes);
int hgt_edge_backward_dst(const float* q, const float* kv, const float* kvr, const float* agg, const float* dagg,
                          const float* stats, const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                          const int32_t* tiles, int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs,
                          int64_t n_nodes, int32_t d, int32_t n_heads, float* dq, float* D,
                          void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_rows(const float* q, const float* dagg, const float* stats, const float* D, const float* own,
                           const float* oth, const int32_t* src_ptr, const int32_t* src_dst, const int32_t* src_oth,
                           int32_t n_rows, int64_t own_rows_total, const int32_t* tiles, int32_t n_tiles,
                           int32_t n_split, const int32_t* hubs, int32_t n_hubs, int32_t d, int32_t n_heads,
                           float* grad, void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                           void* stream);

/* The edge forward and the three backward passes on bf16 gather tables: kv [rows+1, 2d] and kvr [P*240+1, 2d] (own /
 * oth for the row pass) hold bf16 elements and are widened to fp32 in registers; q, agg, dagg, stats, att and every
 * output and gradient (dq, dkv, dkvr, grad, D) stay fp32 in the layouts of the fp32 calls.  Arguments, workspaces,
 * supported shapes and the TMA / LDG choice (row bytes, now 4d, % 16) as for the fp32 calls. */
int hgt_edge_forward_bf16(const float* q, const void* kv, const void* kvr,
                          const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                          const int32_t* csr_eid, const int32_t* tiles, int32_t n_tiles, int32_t n_split_tiles,
                          const int32_t* hubs, int32_t n_hubs,
                          int64_t n_nodes, int64_t n_edges, int32_t d, int32_t n_heads, int32_t apply_gelu,
                          float* agg_out, float* att_out, float* stats_out, void* g_hi, void* g_lo,
                          void* workspace, size_t workspace_bytes, int32_t variant, const int32_t* d_tile_counts,
                          const int32_t* type_row0, int32_t num_types, const int32_t* type_active, void* stream);
/* The edge forward on 24-bit gather tables (see hgt_typed_linear_t24): kv [rows+1] and kvr [P*240+1] rows of 6d bytes,
 * decoded to fp32 in registers; everything else as hgt_edge_forward_bf16.  Needs d % 8 == 0.  There is no backward:
 * training keeps fp32 (or bf16) tables. */
int hgt_edge_forward_t24(const float* q, const void* kv, const void* kvr,
                         const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                         const int32_t* csr_eid, const int32_t* tiles, int32_t n_tiles, int32_t n_split_tiles,
                         const int32_t* hubs, int32_t n_hubs,
                         int64_t n_nodes, int64_t n_edges, int32_t d, int32_t n_heads, int32_t apply_gelu,
                         float* agg_out, float* att_out, float* stats_out, void* g_hi, void* g_lo,
                         void* workspace, size_t workspace_bytes, int32_t variant, const int32_t* d_tile_counts,
                         const int32_t* type_row0, int32_t num_types, const int32_t* type_active, void* stream);
/* The edge forward on bs16 gather tables (see hgt_typed_linear_bs16): kv [rows+1] and kvr [P*240+1] rows of the bs16
 * row bytes of 2d, decoded to fp32 in registers (each element's m * s, exact), so the result equals hgt_edge_forward's
 * on the decoded tables, bitwise.  Everything else as hgt_edge_forward_bf16.  Needs d % 16 == 0.  No backward. */
int hgt_edge_forward_bs16(const float* q, const void* kv, const void* kvr,
                          const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                          const int32_t* csr_eid, const int32_t* tiles, int32_t n_tiles, int32_t n_split_tiles,
                          const int32_t* hubs, int32_t n_hubs,
                          int64_t n_nodes, int64_t n_edges, int32_t d, int32_t n_heads, int32_t apply_gelu,
                          float* agg_out, float* att_out, float* stats_out, void* g_hi, void* g_lo,
                          void* workspace, size_t workspace_bytes, int32_t variant, const int32_t* d_tile_counts,
                          const int32_t* type_row0, int32_t num_types, const int32_t* type_active, void* stream);
int hgt_edge_backward_bf16(const float* q, const void* kv, const void* kvr, const float* agg, const float* dagg,
                           const float* stats, const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                           const int32_t* tiles, int32_t n_tiles, int64_t n_nodes, int32_t d, int32_t n_heads,
                           int64_t kv_rows_total, int64_t kvr_rows_total,
                           float* dq, float* dkv, float* dkvr, void* workspace, size_t workspace_bytes,
                           const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_dst_bf16(const float* q, const void* kv, const void* kvr, const float* agg, const float* dagg,
                               const float* stats, const int32_t* row_ptr, const int32_t* kv_row,
                               const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles, int32_t n_split,
                               const int32_t* hubs, int32_t n_hubs, int64_t n_nodes, int32_t d, int32_t n_heads,
                               float* dq, float* D, void* workspace, size_t workspace_bytes,
                               const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_rows_bf16(const float* q, const float* dagg, const float* stats, const float* D, const void* own,
                                const void* oth, const int32_t* src_ptr, const int32_t* src_dst,
                                const int32_t* src_oth, int32_t n_rows, int64_t own_rows_total, const int32_t* tiles,
                                int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs, int32_t d,
                                int32_t n_heads, float* grad, void* workspace, size_t workspace_bytes,
                                const int32_t* d_tile_counts, void* stream);

/* Backward with a gradient of att as well (a loss term reads the softmax weights att_out of hgt_edge_forward).  With
 * datt [E,H] in ORIGINAL edge order and p = att:  C_i = sum_{e->i} p_e datt_e,  ds_e = p_e ((dp_e + datt_e) - (D_i + C_i));
 * dq, d[K'|V'] and dkvr follow from ds as in the calls above.  datt = 0 gives bitwise their results.
 * hgt_edge_att_grad_prep: writes c_att [N,H] (rows of destinations the tiles cover) and datt_csr [E,H] = datt permuted to
 *   CSR order (datt_csr[c] = datt[csr_eid[c]]).  att is the forward's att_out.  tiles / n_split / hubs / n_hubs /
 *   d_tile_counts: the edge tiles, as for hgt_edge_forward.  No float atomics (hub pieces summed in piece order), so one
 *   call serves the atomic and the deterministic backward.  workspace: hgt_edge_att_grad_workspace_bytes(n_split, H).
 * hgt_edge_backward_att / _dst_att / _rows_att (+ _bf16): the calls above with datt_csr and c_att (rows pass: datt_csr
 *   and src_pos [E], the CSR position of every entry of the source-major index, in index order, from
 *   hgt_plan_source_index_pos).  The destination pass stores D_i + C_i
 *   into D, which the row pass reads unchanged.  Workspaces as above. */
int hgt_edge_att_grad_workspace_bytes(int32_t n_split, int32_t n_heads, size_t* out_bytes);
int hgt_edge_att_grad_prep(const float* att, const float* datt, const int32_t* csr_eid, const int32_t* row_ptr,
                           const int32_t* tiles, int32_t n_tiles, int32_t n_split, const int32_t* hubs, int32_t n_hubs,
                           int64_t n_nodes, int32_t n_heads, float* c_att, float* datt_csr, void* workspace,
                           size_t workspace_bytes, const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_att(const float* q, const float* kv, const float* kvr, const float* agg, const float* dagg,
                          const float* stats, const float* datt_csr, const float* c_att, const int32_t* row_ptr,
                          const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                          int64_t n_nodes, int32_t d, int32_t n_heads, int64_t kv_rows_total, int64_t kvr_rows_total,
                          float* dq, float* dkv, float* dkvr, void* workspace, size_t workspace_bytes,
                          const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_dst_att(const float* q, const float* kv, const float* kvr, const float* agg, const float* dagg,
                              const float* stats, const float* datt_csr, const float* c_att, const int32_t* row_ptr,
                              const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                              int32_t n_split, const int32_t* hubs, int32_t n_hubs, int64_t n_nodes, int32_t d,
                              int32_t n_heads, float* dq, float* D, void* workspace, size_t workspace_bytes,
                              const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_rows_att(const float* q, const float* dagg, const float* stats, const float* D,
                               const float* datt_csr, const float* own, const float* oth, const int32_t* src_ptr,
                               const int32_t* src_dst, const int32_t* src_oth, const int32_t* src_pos, int32_t n_rows,
                               int64_t own_rows_total, const int32_t* tiles, int32_t n_tiles, int32_t n_split,
                               const int32_t* hubs, int32_t n_hubs, int32_t d, int32_t n_heads, float* grad,
                               void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_att_bf16(const float* q, const void* kv, const void* kvr, const float* agg, const float* dagg,
                               const float* stats, const float* datt_csr, const float* c_att, const int32_t* row_ptr,
                               const int32_t* kv_row, const int32_t* rte_row, const int32_t* tiles, int32_t n_tiles,
                               int64_t n_nodes, int32_t d, int32_t n_heads, int64_t kv_rows_total,
                               int64_t kvr_rows_total, float* dq, float* dkv, float* dkvr, void* workspace,
                               size_t workspace_bytes, const int32_t* d_tile_counts, void* stream);
int hgt_edge_backward_dst_att_bf16(const float* q, const void* kv, const void* kvr, const float* agg, const float* dagg,
                                   const float* stats, const float* datt_csr, const float* c_att,
                                   const int32_t* row_ptr, const int32_t* kv_row, const int32_t* rte_row,
                                   const int32_t* tiles, int32_t n_tiles, int32_t n_split, const int32_t* hubs,
                                   int32_t n_hubs, int64_t n_nodes, int32_t d, int32_t n_heads, float* dq, float* D,
                                   void* workspace, size_t workspace_bytes, const int32_t* d_tile_counts,
                                   void* stream);
int hgt_edge_backward_rows_att_bf16(const float* q, const float* dagg, const float* stats, const float* D,
                                    const float* datt_csr, const void* own, const void* oth, const int32_t* src_ptr,
                                    const int32_t* src_dst, const int32_t* src_oth, const int32_t* src_pos,
                                    int32_t n_rows, int64_t own_rows_total, const int32_t* tiles, int32_t n_tiles,
                                    int32_t n_split, const int32_t* hubs, int32_t n_hubs, int32_t d, int32_t n_heads,
                                    float* grad, void* workspace, size_t workspace_bytes,
                                    const int32_t* d_tile_counts, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of the typed linears (training path).  For the group / column-block tables of the forward call:
 *   dA[a_row0_g + m, k]             = sum_c sum_n dOut_c[m, n] * W[w_row0_g + c*cb_width + n, k]   (* gelu'(gelu_aux) if given)
 *   dW[w_row0_g + c*cb_width + n,k] += sum_m dOut_c[m, n] * A[a_row0_g + m, k]
 *   db[w_row0_g + c*cb_width + n]   += sum_m dOut_c[m, n]           (groups with has_bias)
 * dout has the layout of the forward's `out` (flat buffer addressed through the column-block table, dout_elems
 * elements).  dW / db are ACCUMULATED INTO (several groups may share W rows: the caller zero-initialises them once per
 * step); dA is written (rows BETWEEN / BEFORE the groups that no group covers are zeroed; rows past the last group are the
 * caller's) unless accumulate_dA != 0, in which case the product is added to its current content.  dA / dW / db may each be NULL to skip that product.
 * Tensor-core path (impl 0 = auto, 2 = force): wgmma split-bf16 x3 like the forward; impl 3 = auto with one bf16 product
 * (dout, A and W rounded to bf16; only their hi halves are made, so dout_lo / a_lo may be NULL with a pre-split
 * dout_hi / a_hi, and the workspace is at most impl 2's; db is still summed from the fp32 dout; where auto picks SIMT the
 * result stays fp32 SIMT, except that a pre-split A selects the tensor cores as impl 2 does); any other impl is rejected; takes the operands either as
 * fp32 (split here; the dout split pass also yields db) or already split by their producers (dout_hi/lo in dout's
 * layout; a_hi/a_lo [rows, K] as left by hgt_act_split in the forward) — with a pre-split dout, db is NOT computed.
 * impl 1 = fp32 SIMT kernels (any shape; also chosen automatically for cb_width % 8, K % 16, K < 64, overlapping groups
 * such as the RTE tables, or tiny problems).  h_cblocks: HOST copy of the column-block table.  Any number of groups is
 * accepted: the choice of path is made once over the whole table.  The call enqueues only
 * device work (the host-built tables travel in kernel parameters), so it can be captured in a CUDA graph. */
int hgt_typed_linear_bwd_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                                         int32_t K, int32_t cb_width, int64_t lda, int64_t dout_elems,
                                         int32_t have_dout_split, int32_t have_a_split, int32_t impl, size_t* out_bytes);
int hgt_typed_linear_bwd(const float* dout, const void* dout_hi, const void* dout_lo, int64_t dout_elems,
                         const float* A, int64_t lda, const void* a_hi, const void* a_lo,
                         const float* W, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                         const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                         float* dA, int32_t accumulate_dA, const float* gelu_aux, float* dW, float* db,
                         int32_t impl, void* workspace, size_t workspace_bytes, void* stream);

/* Deterministic twin of hgt_typed_linear_bwd (same arguments and results, no float atomics).  dW: every (column block,
 * row chunk) stores its partial tile into the workspace, and the partials are added to dW in (column block, chunk) order;
 * db: per-CTA partial column sums, added in the same order; SIMT dA: one thread per element, over the covering groups in
 * group order.  The workspace grows by the partial slots: tensor cores ~ (4 * SMs / tiles per block + blocks) slots of
 * cb_width x K floats, SIMT at most ~256 + blocks such slots, plus rows / 256 bias rows of cb_width floats. */
int hgt_typed_linear_bwd_det_workspace_bytes(const hgt_lin_group* h_groups, int32_t n_groups,
                                             const hgt_lin_cblock* h_cblocks, int32_t K, int32_t cb_width, int64_t lda,
                                             int64_t dout_elems, int32_t have_dout_split, int32_t have_a_split,
                                             int32_t impl, size_t* out_bytes);
int hgt_typed_linear_bwd_det(const float* dout, const void* dout_hi, const void* dout_lo, int64_t dout_elems,
                             const float* A, int64_t lda, const void* a_hi, const void* a_lo,
                             const float* W, int32_t K, int32_t cb_width, const hgt_lin_group* groups,
                             const hgt_lin_group* h_groups, int32_t n_groups, const hgt_lin_cblock* h_cblocks,
                             float* dA, int32_t accumulate_dA, const float* gelu_aux, float* dW, float* db,
                             int32_t impl, void* workspace, size_t workspace_bytes, void* stream);

/* dW and db of hgt_typed_linear_bf16a (no dA: a bf16 A takes no gradient), and the deterministic twin.  A is bf16
 * [rows, K] at row stride lda; the other arguments are hgt_typed_linear_bwd's.  The tensor-core path (impl 2, 3, or 0
 * where it would take the tensor cores; it needs lda == K) reads A as the dW product's operand as it is and runs
 * dOut_hi*A + dOut_lo*A (dOut_hi*A at impl 3); the SIMT path widens A as it loads it.  dW and db are bitwise those of
 * the fp32 call (same flag) on the widened A.  Workspace: the fp32 queries with have_a_split = 1. */
int hgt_typed_linear_bwd_bf16a(const float* dout, int64_t dout_elems, const void* A, int64_t lda, int32_t K,
                               int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                               int32_t n_groups, const hgt_lin_cblock* h_cblocks, float* dW, float* db, int32_t impl,
                               void* workspace, size_t workspace_bytes, void* stream);
int hgt_typed_linear_bwd_bf16a_det(const float* dout, int64_t dout_elems, const void* A, int64_t lda, int32_t K,
                                   int32_t cb_width, const hgt_lin_group* groups, const hgt_lin_group* h_groups,
                                   int32_t n_groups, const hgt_lin_cblock* h_cblocks, float* dW, float* db,
                                   int32_t impl, void* workspace, size_t workspace_bytes, void* stream);

/* act(in) as fp32 (out_f32 [rows, K], or NULL) and/or as the bf16 hi/lo operand split (hi/lo [rows, K], or NULL; needs
 * K % 8 == 0; hi without lo writes only the hi half, bitwise the same, the operand of a one-product GEMM).  act: 0 = identity, 1 = exact-erf gelu (conv.py:119).  The training forward keeps the split for the
 * backward pass (it is the A operand of the dW product). */
int hgt_act_split(const float* in, int64_t ld, int64_t rows, int32_t K, int32_t act, float* out_f32,
                  void* hi, void* lo, void* stream);

/* Backward of hgt_update_epilogue (conv.py:129-133).  dout [N,d] in ORIGINAL node order (perm as in the forward);
 * o / x [N,d] rank order (the forward's inputs); norm_w [T,d] or NULL.  Outputs: d_o, d_x [N,d] rank order (rows of
 * out-of-range type get zeros), d_skip [T], d_norm_w / d_norm_b [T,d] (zero-initialised by this call).
 * skip == NULL: residual mode (y = o + x), d_skip is not touched.  type_active as in the forward: rows past
 * type_active[t] get zero gradients and their (never computed) `o` rows are not read. */
int hgt_update_backward(const float* dout, const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                        const float* skip, const float* norm_w, const int32_t* perm, const int32_t* type_active,
                        int64_t n_nodes, int32_t d,
                        float* d_o, float* d_x, float* d_skip, float* d_norm_w, float* d_norm_b, void* stream);
/* Deterministic twin: blocks never cross a type boundary, each stores its d norm / d skip sums in its own workspace slot,
 * and each type's slots are added in block order (no atomics).  Outputs are written, not accumulated. */
int hgt_update_backward_det_workspace_bytes(int64_t n_nodes, int32_t num_types, int32_t d, size_t* out_bytes);
int hgt_update_backward_det(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                            int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                            const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                            float* d_skip, float* d_norm_w, float* d_norm_b, void* workspace, size_t workspace_bytes,
                            void* stream);

/* Backward of hgt_fold_weights for the K'/V' blocks: from d W_cat / d b_cat to the gradients of k_linears / v_linears
 * (stacked [T, d_out, d_in] / [T, d_out]) and relation_att / relation_msg [R,H,dk,dk], relation_pri [R,H]; all outputs
 * are zero-initialised by this call.  (The W_q rows of W_cat are plain copies: their gradient is the matching slice.) */
int hgt_fold_backward(const float* d_w_cat, const float* d_b_cat, const float* const* wk, const float* const* bk,
                      const float* const* wv, const float* const* bv, const float* relation_att,
                      const float* relation_msg, const float* relation_pri, int32_t num_types, int32_t num_relations,
                      int32_t n_heads, int32_t d_in, int32_t d_out, int32_t n_pairs, const int32_t* pair_type,
                      const int32_t* pair_rel, const int32_t* cat_row0, float* d_wk, float* d_bk, float* d_wv,
                      float* d_bv, float* d_att, float* d_msg, float* d_pri, void* stream);
/* Deterministic twin: every output element is computed by one thread (warp for the relation matrices), which loops over
 * the <type, relation> pairs in pair order.  Same arguments and results. */
int hgt_fold_backward_det(const float* d_w_cat, const float* d_b_cat, const float* const* wk, const float* const* bk,
                          const float* const* wv, const float* const* bv, const float* relation_att,
                          const float* relation_msg, const float* relation_pri, int32_t num_types, int32_t num_relations,
                          int32_t n_heads, int32_t d_in, int32_t d_out, int32_t n_pairs, const int32_t* pair_type,
                          const int32_t* pair_rel, const int32_t* cat_row0, float* d_wk, float* d_bk, float* d_wv,
                          float* d_bv, float* d_att, float* d_msg, float* d_pri, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Update epilogue (conv.py:129-133): y = o*sigmoid(skip[t]) + x*(1-sigmoid(skip[t])); LayerNorm_t(y)
 * (eps 1e-5, affine) iff use_norm; rows of out-of-range type are written as zeros (conv.py:120).
 * skip == NULL selects the plain residual y = o + x of DenseHGTConv (conv.py:261,273).
 *   o [N,d] rank order (a_linear output, after dropout if training);  x [N,d] rank order;
 *   type_row0 [T+2] int32 prefix of type_count;  norm_w/norm_b [T,d] or NULL;  perm NULL if identity;
 *   type_active [T] int32 or NULL: when given, only the first type_active[t] rows of type t are written
 *   (sharded runs: the remaining rows are halo sources that need no output);
 *   out [N,d] in ORIGINAL node order;
 *   out_hi / out_lo [N,d] bf16 or NULL: `out` again as the bf16 hi/lo split that the NEXT layer's projection GEMM
 *   consumes (hgt_typed_linear_presplit) — only with perm == NULL, type_active == NULL, d % 8 == 0; out_hi without
 *   out_lo writes the hi half only (for a one-product GEMM).
 * ---------------------------------------------------------------------------------------------- */
int hgt_update_epilogue(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                        const float* skip, const float* norm_w, const float* norm_b,
                        const int32_t* perm, const int32_t* type_active, int64_t n_nodes, int32_t d,
                        float* out, void* out_hi, void* out_lo, void* stream);
/* hgt_update_epilogue without type_active, for a layer whose a_linear covered only the first type_dst[t] rows of every
 * type t (type_dst [T] int32, the extents of hgt_plan_dst_end): the other rows have no in-edges, so their a_linear
 * output is exactly the bias, and they read o = bias[t] ([T, d], the a_linears' biases) instead of their `o` row, which
 * is never read.  Every row is written, as by hgt_update_epilogue. */
int hgt_update_epilogue_dst(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                            const float* skip, const float* norm_w, const float* norm_b, const int32_t* perm,
                            const int32_t* type_dst, const float* bias, int64_t n_nodes, int32_t d, float* out,
                            void* out_hi, void* out_lo, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Fused dropout: training dropout drawn inside the kernels, nothing stored.
 *
 * Mask contract.  Element (row, col) of an [N, d] tensor is kept iff word (col % 4) of
 *     Philox4x32-10(counter = (q_lo32, q_hi32, 0, 0), key = (seed_lo32, seed_hi32)),   q = row * ceil(d / 4) + col / 4
 * is >= thr, thr = (uint32)((double)p * 2^32) with p the fp32 value passed.  `row` is the kernel's rank-order row (never
 * perm[row]); `seed` is ONE 64-bit value read from DEVICE memory by the kernel (no host read-back, so a captured CUDA
 * graph draws new masks whenever the seed buffer is rewritten).  Philox4x32-10 is the raw ten-round block function
 * (curand_Philox4x32_10): no generator state, no curand_init.  Kept values are multiplied by s = 1 / (1 - p) in fp32;
 * p >= 1 drops every element (s = 0); p <= 0 is refused.  The mask therefore depends on (seed, row, col, d, p) alone: not
 * on the launch geometry, the vector or scalar kernel instance, perm / type_active, or the deterministic twin.  A
 * backward kernel given the same (seed, p) regenerates the forward's mask bit for bit.
 *
 * hgt_update_epilogue_drop: hgt_update_epilogue with o <- o * mask * s applied as the row is loaded.  Rows that are not
 *   written (type_active, perm < 0) or are written as zeros (unknown type) draw nothing.  There is no type_dst form (that
 *   table belongs to inference).  out_hi / out_lo as in hgt_update_epilogue.
 * hgt_update_backward_drop[_det]: hgt_update_backward[_det] for that forward.  `o` is the PRE-dropout tensor the forward
 *   read; the kernels use o * mask * s wherever the plain ones use o (LayerNorm recompute, d skip) and store
 *   d o * mask * s.  The _det form takes the workspace of hgt_update_backward_det_workspace_bytes.
 * hgt_tanh_dropout: out = tanh(x) * mask * s over the first n_rows of [n_total, d]; rows past n_rows (nodes of unknown
 *   type) are copied unchanged.  out may alias x.
 * hgt_tanh_dropout_bwd: d_x = dout * mask * s * (1 - tanh(x)^2) from `out` alone (where the mask is 1, tanh(x) = out / s;
 *   elsewhere the gradient is 0); rows past n_rows: d_x = dout.  d_x may alias dout.
 * ---------------------------------------------------------------------------------------------- */
int hgt_update_epilogue_drop(const float* o, const float* x, const int32_t* type_row0, int32_t num_types,
                             const float* skip, const float* norm_w, const float* norm_b, const int32_t* perm,
                             const int32_t* type_active, int64_t n_nodes, int32_t d, float* out, void* out_hi,
                             void* out_lo, const uint64_t* seed, float p, void* stream);
int hgt_update_backward_drop(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                             int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                             const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                             float* d_skip, float* d_norm_w, float* d_norm_b, const uint64_t* seed, float p,
                             void* stream);
int hgt_update_backward_drop_det(const float* dout, const float* o, const float* x, const int32_t* type_row0,
                                 int32_t num_types, const float* skip, const float* norm_w, const int32_t* perm,
                                 const int32_t* type_active, int64_t n_nodes, int32_t d, float* d_o, float* d_x,
                                 float* d_skip, float* d_norm_w, float* d_norm_b, void* workspace,
                                 size_t workspace_bytes, const uint64_t* seed, float p, void* stream);
int hgt_tanh_dropout(const float* x, int64_t n_rows, int64_t n_total, int32_t d, const uint64_t* seed, float p,
                     float* out, void* stream);
int hgt_tanh_dropout_bwd(const float* dout, const float* out, int64_t n_rows, int64_t n_total, int32_t d,
                         const uint64_t* seed, float p, float* d_x, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Whole layer in one call (inference): HGTConv.forward, pyHGT/conv.py:56-134.
 * Every pointer below is a DEVICE pointer except the h_* tables (host copies of the typed-linear group tables, used
 * only to size grids).  Parameter pointer tables (wq ... norm_b) are device arrays of num_types device pointers, one
 * per nn.Linear / nn.LayerNorm of the module (conv.py:34-40).  The plan arrays come from hgt_plan_*; the typed-linear
 * tables are the ones hgt_typed_linear takes (projection: Q + [K'|V'] blocks; rte: K'R/V'R tables; rt: the single
 * 240 x d group of RelTemporalEncoding.lin; upd: a_linears).  Nothing is allocated or synchronised.
 * The [K'|V'] and RTE tables take the format hgt_gather_table_format picks for the device's L2: bs16
 * (hgt_typed_linear_bs16, hgt_edge_forward_bs16), 24-bit (hgt_typed_linear_t24, hgt_edge_forward_t24) or fp32.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  /* sizes and switches */
  int64_t n_nodes, n_edges, kv_rows, cat_rows, q_off, kv_off, proj_elems;
  int32_t num_types, num_relations, n_heads, d_in, d_out, n_pairs;
  int32_t use_rte, use_norm, edge_variant;
  int32_t linear_impl;        /* hgt_typed_linear's impl for the projection and a_linear GEMMs; 3: one bf16 product, then
                                 the edge kernel's operand split is hi only and x_lo is not read */
  int32_t n_tiles, n_split, n_hubs;
  int32_t n_proj_groups, n_rte_groups, n_upd_groups;
  /* plan (hgt_plan_*) */
  const int32_t* perm;        /* NULL when node_type is already sorted */
  const int32_t* type_row0;   /* [T+2] */
  const int32_t* type_active; /* [T] or NULL (sharded runs) */
  const int32_t* out_map;     /* [N] or NULL: rank-order row -> output row (sharded runs) */
  const int32_t* row_ptr;
  const int32_t* kv_row;
  const int32_t* rte_row;     /* NULL when !use_rte */
  const int32_t* csr_eid;
  const int32_t* tiles;
  const int32_t* hubs;
  const int32_t* d_tile_counts; /* NULL, or device {n_tiles, n_split, n_hubs}: n_tiles/n_split/n_hubs above are bounds */
  const int32_t* pair_type;
  const int32_t* pair_rel;
  const int32_t* cat_row0;
  const int32_t* q_row0;
  /* typed-linear tables */
  const hgt_lin_group* proj_groups; const hgt_lin_group* h_proj_groups; const hgt_lin_cblock* proj_cblocks;
  const hgt_lin_group* rte_groups;  const hgt_lin_group* h_rte_groups;  const hgt_lin_cblock* rte_cblocks;
  const hgt_lin_group* rt_groups;   const hgt_lin_group* h_rt_groups;   const hgt_lin_cblock* rt_cblocks;
  const hgt_lin_group* upd_groups;  const hgt_lin_group* h_upd_groups;  const hgt_lin_cblock* upd_cblocks;
  /* parameters */
  const float* const* wq; const float* const* bq;
  const float* const* wk; const float* const* bk;
  const float* const* wv; const float* const* bv;
  const float* const* wa; const float* const* ba;
  const float* const* norm_w; const float* const* norm_b;   /* NULL when !use_norm; the vectors may sit at any float
                                                               alignment (e.g. views into one flat parameter buffer) */
  const float* relation_att; const float* relation_msg; const float* relation_pri; const float* skip;
  const float* emb_weight; const float* emb_lin_w; const float* emb_lin_b;   /* NULL when !use_rte */
  /* data */
  const float* x;             /* [N, d_in] in original node order */
  const void* x_hi; const void* x_lo;   /* optional: x already split to bf16 hi/lo (rank order == original order) */
  float* out;                 /* [N or out rows, d_out] */
  float* att;                 /* [E, H] or NULL */
  void* out_hi; void* out_lo; /* optional: out again as the bf16 hi/lo split for the next layer */
  const int32_t* type_dst;    /* [T] or NULL: extents of hgt_plan_dst_end (not with type_active).  The proj and upd tables
                                 then hold Q and a_linear rows for the first type_dst[t] rows of each type only; the other
                                 rows have no in-edges and take the a_linear bias (hgt_update_epilogue_dst) */
} hgt_conv_args;

uint64_t hgt_conv_args_size(void);   /* sizeof(hgt_conv_args): lets a foreign-language binding check its struct layout */
int hgt_conv_workspace_bytes(const hgt_conv_args* args, size_t* out_bytes);
int hgt_conv_forward(const hgt_conv_args* args, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * HOST helper of HGSampling (pyHGT/data.py:123-130; pyhgt_b200/sampler.py): every pointer is a HOST pointer, nothing
 * touches the GPU.  Applies the sampled neighbours of one <target type, source type, relation> adjacency slice to the
 * budget of the source type (flat arrays over node ids; `stamp` reproduces the reference dict's insertion order).
 * Returns the number of budget entries added / updated, -1 if an id lies outside [0, n). */
int64_t hgt_sampler_budget_update(const int64_t* h_ids, const int64_t* h_times, int64_t n_sampled, int64_t target_time,
                                  int64_t no_time, int64_t max_time, int64_t n, const uint8_t* h_in_layer,
                                  uint8_t* h_in_budget, double* h_score, int64_t* h_budget_time, int64_t* h_stamp,
                                  int64_t* h_stamp_counter, int32_t* h_touched_layer);

/* Bits of the `skip` word of hgt_sampler_block and hgt_gsample_block.  HGT_BLOCK_SKIP marks the 'self' relation
 * (data.py:116), as the value 1 always has.  HGT_BLOCK_NARROW marks a block whose row_of / ptr / nbr / time arrays are
 * int32 instead of int64 (the pointers keep their int64_t* type and are read as int32_t*); in its time array INT32_MIN
 * stands for no_time (the reference's `None`).  A word of 0 or 1, which is all earlier callers pass, is the int64 layout.
 * The flag rides in `skip` so that the structs keep their size: callers allocate arrays of them. */
#define HGT_BLOCK_SKIP 1
#define HGT_BLOCK_NARROW 2

/* One <target type, source type, relation> adjacency of the frozen graph in CSR form (host arrays; rows in the
 * reference dict's insertion order) and the layer_data / budget of one node type as flat arrays over node ids. */
typedef struct {
  const int64_t* row_of; int64_t n_row_of;   /* target id -> CSR row, -1 = no adjacency */
  const int64_t* ptr; const int64_t* nbr; const int64_t* time;
  int32_t src_state;                         /* index of the source type's hgt_sampler_state */
  int32_t skip;                              /* HGT_BLOCK_SKIP for the 'self' relation, | HGT_BLOCK_NARROW (see above) */
} hgt_sampler_block;
typedef struct {
  int64_t n;
  uint8_t* in_layer; uint8_t* in_budget; double* score; int64_t* b_time; int64_t* stamp;
  int64_t* log; int64_t log_len;             /* ids in budget-insertion order (capacity n) */
  int64_t layer_seq; int64_t budget_seq;     /* first-touch numbers of layer_data[type] / budget[type], -1 = untouched */
} hgt_sampler_state;
/* add_budget (pyHGT/data.py:108-130) for a batch of target nodes of one type, target-major, blocks in dict order; the
 * uniform draws are made by the caller (numpy's global RNG, same order) and passed as positions.  0 = ok. */
int64_t hgt_sampler_add_budget(const int64_t* h_target_ids, const int64_t* h_target_times, int64_t n_targets,
                               const hgt_sampler_block* h_blocks, int32_t n_blocks, hgt_sampler_state* h_states,
                               int32_t n_states, int64_t sampled_number, const int64_t* h_draw_off,
                               const int64_t* h_draw_pos, int64_t no_time, int64_t max_time, int64_t* h_counters);

/* ------------------------------------------------------------------------------------------------
 * HGSampling on the GPU (pyHGT/data.py:87-256; pyhgt_b200/sampler.py: sample_subgraph_cuda).  Same distribution over
 * sampled node sets, times and order as the host sampler, drawn with Philox (seed, step) streams instead of numpy's;
 * bitwise repeatable for a given seed.  A batch runs: rows of the seeds written by the caller, add_budget for the seeds
 * of every seed type, then per sampling layer and type select + add_budget, then rebuild_count -> (read back) ->
 * rebuild_write.  Node types are numbered 0..T-1 ("slots"); the node with id `i` of type t is state slot type_off[t]+i.
 * ---------------------------------------------------------------------------------------------- */

/* One <target type, source type, relation> adjacency in CSR form, rows in the reference dict's insertion order.  The
 * struct itself lives in DEVICE memory (an array of them per call); the arrays it points to are device memory or
 * device-mapped page-locked host memory (hgt_host_register). */
typedef struct {
  const int64_t* row_of; int64_t n_row_of;   /* target id -> CSR row, -1 = no adjacency */
  const int64_t* ptr;                         /* [rows+1] positions into nbr / time */
  const int64_t* nbr; const int64_t* time;    /* neighbour ids and edge times in dict order (no_time = None) */
  int32_t tgt_type, src_type;                 /* type slots */
  int32_t skip;                               /* HGT_BLOCK_SKIP for the 'self' relation: never sampled from
                                                 (data.py:116); | HGT_BLOCK_NARROW: the four arrays are int32 */
  int32_t rel;                                /* edge_type value in the to_torch layout (data.py:237-238) */
} hgt_gsample_block;

/* ------------------------------------------------------------------------------------------------
 * B subgraphs ("members") in one pass (pyhgt_b200/sampler.py: sample_subgraphs_cuda; sample_subgraph_cuda is B = 1).
 * The members share the graph, the time filter, the depth and the width; each has its own seeds, Philox seed, step
 * numbers and rows of the state, and member b's result is bitwise that of a batch of b alone with the same seed and
 * steps.  Memory: about 52 bytes per state slot, i.e. B x 52 B x (sum of the id ranges) for the dense arrays; selection
 * sorts every id of the selected type (int32 sort values: the ranges of one step must sum to less than 2^31 - 1).  The
 * hashed state below (hgt_gsample_hash_state) holds the same fields in hash tables sized by the sample instead.
 * ---------------------------------------------------------------------------------------------- */

/* Dense sampler state of B members: the struct is passed by HOST pointer, its fields are DEVICE arrays.  type_off /
 * lid_off hold ABSOLUTE positions (member b's type t: slots type_off[b*(T+1)+t] .. [b*(T+1)+t+1], lid entries likewise);
 * the per-slot arrays hold every member's slots.  Initial values, per member: ser -1, n_layer 0, score 0, bstamp -1,
 * last_seq -1, first_seq / type_min INT64_MAX, type_seq -1 (except the seed types' layer numbers), counters {number of
 * seed types, 0}. */
typedef struct {
  int32_t num_types; int32_t n_members;
  const int64_t* type_off;   /* [B*(T+1)] first state slot of each (member, type) (id range: the difference to the next) */
  const int64_t* lid_off;    /* [B*(T+1)] first entry of each (member, type) in lid (capacity: likewise) */
  int32_t* ser;              /* [slots] position of the node in layer_data[type] (data.py:133-141,166), -1 = not sampled */
  int64_t* ltime;            /* [slots] its time in layer_data */
  int64_t* lid;              /* sampled ids of every (member, type) in ser order */
  int64_t* n_layer;          /* [B*T] nodes sampled per type */
  unsigned long long* score; /* [slots] budget score, fixed point with 40 fraction bits */
  int64_t* btime;            /* [slots] budget time (last writer, data.py:130) */
  int64_t* bstamp;           /* [slots] budget insertion stamp, -1 = not in the budget */
  int64_t* last_seq;         /* [slots] scratch */
  int64_t* first_seq;        /* [slots] scratch */
  int64_t* type_min;         /* [B*2T] scratch */
  int64_t* type_seq;         /* [B*2T] first-touch number of layer_data[t] (2t) and budget[t] (2t+1), -1 = untouched */
  int64_t* counters;         /* [B*2] next first-touch numbers */
  const uint64_t* seed;      /* [B] each member's Philox seed */
} hgt_gsample_batch_state;

/* add_budget (data.py:108-130) for every member at once: member b's targets are tgt_id / tgt_time [b*max_targets ...]
 * (n_targets[b] of them, device) of node type type[b] (device [B]; -1 = the member sits this step out), whose blocks are
 * blocks[type_blocks[2t] .. type_blocks[2t+1]) (device [2T], dict order; max_blocks >= every such count; non-'self'
 * blocks are sampled).  time_filter = 0 disables the max_time test (ogbn-mag variant: time_range=None).  step [B]
 * (device): the member's step number, unique to this call within the member's run (< 2^22); it selects the random
 * stream and orders the insertion stamps.  flags[0] is set when a neighbour id lies outside its type's id range. */
int hgt_gsample_batch_add_budget_workspace_bytes(int32_t n_members, int64_t max_targets, int32_t max_blocks,
                                                 int64_t sampled_number, size_t* out_bytes);
int hgt_gsample_batch_add_budget(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                 const int32_t* type_blocks, int32_t max_blocks, const int32_t* type, const int64_t* step,
                                 const int64_t* tgt_id, const int64_t* tgt_time, int64_t max_targets,
                                 const int64_t* n_targets, int64_t sampled_number, int32_t time_filter, int64_t max_time,
                                 int64_t no_time, int32_t* flags, void* workspace, size_t workspace_bytes, void* stream);

/* Selection of one (layer, type) per member (data.py:150-170): member b selects from type[b] (-1 = none: n_targets[b] =
 * 0) with step[b].  Every budget entry in insertion order when the budget holds fewer than sampled_number entries, else
 * sampled_number entries without replacement with p ~ score^2 (ordered); they join the layer, leave the budget, and go
 * to tgt_id / tgt_time [b*sampled_number ...] with their count in n_targets[b] (device), ready for add_budget.  Member
 * b's ids are sorted at positions sel_off[b] .. sel_off[b+1] (device [B+1], = the type's id range; n_total =
 * sel_off[B], max_ids >= every range).  flags[0]: layer capacity exceeded. */
int hgt_gsample_batch_select_workspace_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes);
int hgt_gsample_batch_select(const hgt_gsample_batch_state* h_state, const int32_t* type, const int64_t* step,
                             const int64_t* sel_off, int64_t n_total, int64_t max_ids, int64_t sampled_number,
                             int64_t* tgt_id, int64_t* tgt_time, int64_t* n_targets, int32_t* flags, void* workspace,
                             size_t workspace_bytes, void* stream);

/* Rebuild of the sampled adjacency (data.py:190-209), pass 1: for every member b, block k (all relations, 'self'
 * included) and sampled target r of its type, the number of neighbours in the sample, at cnt_off[b*n_blocks+k] + r
 * (cnt_off [B*n_blocks+1]: room for the lid capacity of the target type; n_count = cnt_off[B*n_blocks]).  ex
 * [n_count+1]: exclusive prefix of those counts; totals [B*n_blocks]: edges per (member, block).  max_rows >= every
 * lid capacity.  flags[1]: an edge_time outside [0, 240) (data.py:250, RelTemporalEncoding size); flags[2]: a sampled
 * id >= feat_rows[type] (feat_rows [T] or NULL).  Workspace: hgt_gsample_rebuild_workspace_bytes(n_count), the same for
 * every rebuild count pass (dense, hashed and host-graph).
 * min_ser: NULL (no mask) or an edge mask [2*n_blocks] (device, sampler.py: sample_subgraphs_cuda(..., edge_mask=...))
 * shared by every member: an edge of block k is kept iff its target ser >= min_ser[2k] and its source ser >=
 * min_ser[2k+1]; {0, 0} keeps the whole block.  Pass the same table to both passes: totals and the edge layout then
 * count kept edges only, in block order, and the edge_time check (flags[1]) looks at kept edges only.  The neighbour id
 * check (flags[0]) covers every edge. */
int hgt_gsample_rebuild_workspace_bytes(int64_t n_count, size_t* out_bytes);
int hgt_gsample_batch_rebuild_count(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                    int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off, int64_t n_count,
                                    int64_t max_rows, const int64_t* feat_rows, int64_t* ex, int64_t* totals,
                                    int32_t* flags, void* workspace, size_t workspace_bytes, void* stream);
/* Pass 2: the to_torch layout (data.py:226-256) of every member.  Member-local tables: node_off [B*T]: first output row
 * of each type (-1 = not laid out), type_out [T]: its node_type value; self_off [B*T]: first edge of its self loops (-1
 * = none), blk_out [B*n_blocks]: first edge of each block's edges (-1 = none).  mem_out [B*4] (device): member b's
 * {first node row, first edge, position of its first source, position of its first destination} in the shared outputs
 * (four columns since the fixed-shape sampler below: before it, three, {first node row, first edge, edge count}):
 * its edge e has edge_type / edge_time at first edge + e and edge_index[src + e] / [dst + e].  edge_type / edge_time
 * [edges], node_type / node_time [rows].  Node ids in edge_index are node_off + ser (without the first node row):
 * sample_subgraphs_cuda passes {node_base, edge_base, 2 * edge_base, 2 * edge_base + E_b}, so that member b's
 * edge_index is the [2, E_b] block at edge_index + 2 * edge_base with member-local ids, exactly a to_torch layout.  node_feature [rows, feat_dim] gathered from feat[t]
 * (a DEVICE array of T device pointers to [ids, feat_dim] float tables) or NULL. */
int hgt_gsample_batch_rebuild_write(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                    int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off, const int64_t* ex,
                                    const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
                                    const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows,
                                    const float* const* feat, int32_t feat_dim, int64_t* node_type, int64_t* node_time,
                                    float* node_feature, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time,
                                    void* stream);

/* The hashed sampler state (sampler.py: sample_subgraphs_cuda picks it when the dense state is too large or slower):
 * per (member, type) an open-addressing table of `room` entries keyed by node id, sized by the sample rather than by the
 * id range.  Results are bitwise those of the dense state for the same inputs.
 *   ent_off [B*(T+1)]: ABSOLUTE first entry of each (member, type) region (member b's type t: entries ent_off[b*(T+1)+t]
 *     .. [b*(T+1)+t+1]); lid_off as for hgt_gsample_batch_state; n_ids [B*T]: the id range of each (member, type)
 *     (neighbour ids outside it set flags[0], as in the dense state; ids must stay below 2^40).
 *   key [entries]: node id of the entry, -1 = empty (every entry starts empty); ser / score / btime / bstamp /
 *     last_seq / first_seq [entries]: the dense per-slot fields with the dense initial values.
 *   ltime [lid entries]: the time of every sampled node, indexed like lid (per ser, not per id).
 *   fill [B*T]: entries claimed per region, initially 0.  n_layer, type_min, type_seq, counters, seed: as dense.
 * An entry is claimed with one compare-and-swap on its key; probing is linear and visits a region at most once.  A claim
 * that takes a region past half full, or finds no free entry, sets flags[3] (overflow): the results of that run are
 * incomplete and it must be repeated with larger regions.  Nothing is written outside the regions. */
typedef struct {
  int32_t num_types; int32_t n_members;
  const int64_t* ent_off;
  const int64_t* lid_off;
  const int64_t* n_ids;
  int64_t* key;
  int32_t* ser;
  int64_t* ltime;
  int64_t* lid;
  int64_t* n_layer;
  unsigned long long* score;
  int64_t* btime;
  int64_t* bstamp;
  int64_t* last_seq;
  int64_t* first_seq;
  unsigned long long* fill;
  int64_t* type_min;
  int64_t* type_seq;
  int64_t* counters;
  const uint64_t* seed;
} hgt_gsample_hash_state;

/* The seeds (data.py:135-137): seed i of region[i] = b*T + t (device arrays [n]) gets an entry for id[i] with ser[i],
 * and lid / ltime at position ser[i] of that (member, type).  region[i] < 0: no seed (padding of a fixed-size table). */
int hgt_gsample_hash_insert_seeds(const hgt_gsample_hash_state* h_state, int64_t n, const int64_t* region,
                                  const int64_t* id, const int64_t* ser, const int64_t* time, int32_t* flags,
                                  void* stream);
/* As hgt_gsample_batch_add_budget (same arguments, same workspace: hgt_gsample_batch_add_budget_workspace_bytes). */
int hgt_gsample_hash_add_budget(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                const int32_t* type_blocks, int32_t max_blocks, const int32_t* type, const int64_t* step,
                                const int64_t* tgt_id, const int64_t* tgt_time, int64_t max_targets,
                                const int64_t* n_targets, int64_t sampled_number, int32_t time_filter, int64_t max_time,
                                int64_t no_time, int32_t* flags, void* workspace, size_t workspace_bytes, void* stream);
/* As hgt_gsample_batch_select, over the selected type's REGION instead of its id range: sel_off [B+1] (device) are
 * prefix sums of the region sizes (max_room >= every region size).  The budget entries are ordered by id first, so keys
 * and ties are exactly those of the dense selection.  n_total (< 2^31 - 1) is the number of sorted positions: sel_off[B],
 * or, when the regions are chosen on the device, an upper bound of it up to B * max_room; the positions past sel_off[B]
 * are padding that sorts behind every entry, and the selection is the one n_total = sel_off[B] makes. */
int hgt_gsample_hash_select_workspace_bytes(int32_t n_members, int64_t n_total, size_t* out_bytes);
int hgt_gsample_hash_select(const hgt_gsample_hash_state* h_state, const int32_t* type, const int64_t* step,
                            const int64_t* sel_off, int64_t n_total, int64_t max_room, int64_t sampled_number,
                            int64_t* tgt_id, int64_t* tgt_time, int64_t* n_targets, int32_t* flags, void* workspace,
                            size_t workspace_bytes, void* stream);
/* The rebuild passes, as hgt_gsample_batch_rebuild_count / _write (min_ser included), and the host-graph passes as
 * hgt_gsample_batch_rebuild_count_host / _write_host.  Workspace: hgt_gsample_rebuild_workspace_bytes.  The outputs
 * are those of the dense state. */
int hgt_gsample_hash_rebuild_count(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                   int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off, int64_t n_count,
                                   int64_t max_rows, const int64_t* feat_rows, int64_t* ex, int64_t* totals,
                                   int32_t* flags, void* workspace, size_t workspace_bytes, void* stream);
int hgt_gsample_hash_rebuild_write(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                   int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off, const int64_t* ex,
                                   const int64_t* blk_out, const int64_t* node_off, const int64_t* type_out,
                                   const int64_t* self_off, int64_t self_rel, const int64_t* mem_out, int64_t max_rows,
                                   const float* const* feat, int32_t feat_dim, int64_t* node_type, int64_t* node_time,
                                   float* node_feature, int64_t* edge_index, int64_t* edge_type, int64_t* edge_time,
                                   void* stream);
int hgt_gsample_hash_rebuild_count_host(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                        int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                        int64_t n_count, int64_t max_rows, const int64_t* feat_rows, void* hits,
                                        int64_t hit_cap, int64_t* n_hits, int64_t* ex, int64_t* totals, int32_t* flags,
                                        void* workspace, size_t workspace_bytes, void* stream);
int hgt_gsample_hash_rebuild_write_host(const hgt_gsample_hash_state* h_state, const hgt_gsample_block* blocks,
                                        int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                        const int64_t* ex, const int64_t* blk_out, const int64_t* node_off,
                                        const int64_t* type_out, const int64_t* self_off, int64_t self_rel,
                                        const int64_t* mem_out, int64_t max_rows, const void* hits, int64_t n_hits,
                                        const float* const* feat, int32_t feat_dim, int64_t* node_type,
                                        int64_t* node_time, float* node_feature, int64_t* edge_index,
                                        int64_t* edge_type, int64_t* edge_time, void* stream);

/* Graphs in page-locked host memory (sampler.py: DeviceGraph(..., placement="host")).  hgt_host_register page-locks
 * [host, host + bytes) (cudaHostRegister, mapped) and returns in *dev_ptr the address device code reads it at;
 * hgt_host_unregister undoes it once no kernel reads the range any more.  Blocks whose row_of / ptr / nbr / time are
 * such addresses work with every sampler entry point (the kernels read them in place); the two rebuild passes below are
 * the ones meant for them: the count pass reads each sampled target's neighbour list once and leaves one 16-byte hit
 * record per kept edge in `hits` (device, room for hit_cap < 2^31 records), with their number in *n_hits (device; it
 * counts past hit_cap).  The write pass lays the edges out from the n_hits records alone, or, with hits NULL (the records
 * did not fit), re-reads the lists like hgt_gsample_batch_rebuild_write; it gathers feature rows (feat may point to host
 * tables) with 16-byte loads when they are 16-byte aligned.  Otherwise, min_ser included, as
 * hgt_gsample_batch_rebuild_count / _write: the outputs are identical. */
int hgt_host_register(void* host, size_t bytes, void** dev_ptr);
int hgt_host_unregister(void* host);
int hgt_gsample_batch_rebuild_count_host(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                         int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                         int64_t n_count, int64_t max_rows, const int64_t* feat_rows, void* hits,
                                         int64_t hit_cap, int64_t* n_hits, int64_t* ex, int64_t* totals, int32_t* flags,
                                         void* workspace, size_t workspace_bytes, void* stream);
int hgt_gsample_batch_rebuild_write_host(const hgt_gsample_batch_state* h_state, const hgt_gsample_block* blocks,
                                         int32_t n_blocks, const int64_t* min_ser, const int64_t* cnt_off,
                                         const int64_t* ex, const int64_t* blk_out, const int64_t* node_off,
                                         const int64_t* type_out, const int64_t* self_off, int64_t self_rel,
                                         const int64_t* mem_out, int64_t max_rows, const void* hits, int64_t n_hits,
                                         const float* const* feat, int32_t feat_dim, int64_t* node_type,
                                         int64_t* node_time, float* node_feature, int64_t* edge_index,
                                         int64_t* edge_type, int64_t* edge_time, void* stream);

/* Feature rows from bf16 tables (sampler.py: DeviceGraph(..., feature_dtype=torch.bfloat16)), run after a rebuild write
 * pass that was given feat = NULL: node_feature[i, :] = the widening to float of feat[row_type[i]][row_id[i], :] for the
 * n_rows output rows (a row with row_id[i] < 0 is left as it is).  feat is a DEVICE array of per-type pointers to [ids, feat_dim] bf16 tables (device memory or
 * device-mapped host memory), row_type / row_id [n_rows] DEVICE arrays (a row's type slot and sampled id: the batch's
 * node_type and the sampled ids in output order).  Reads 16 bytes at a time where a row is 16-byte aligned, element by
 * element elsewhere.  Ids are not range-checked here: the rebuild count pass checks them against feat_rows. */
int hgt_gsample_gather_features_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                                     const int64_t* row_id, int64_t n_rows, float* node_feature, void* stream);
/* The same rows kept in bf16 (sample_subgraph(s)_cuda(..., feature_dtype=torch.bfloat16)): node_feature is bf16
 * [n_rows, feat_dim] and each row is copied as stored.  Loads as above; stores take 16 bytes where the output row is
 * 16-byte aligned at that point, 4 or 2 bytes where it is not. */
int hgt_gsample_gather_rows_bf16(const uint16_t* const* feat, int32_t feat_dim, const int64_t* row_type,
                                 const int64_t* row_id, int64_t n_rows, void* node_feature, void* stream);

/* Sampling with fixed shapes and no read-back (sampler.py: GraphedSampler): the host decisions of
 * sample_subgraphs_cuda made on the device, so that a whole call can be captured in a CUDA graph.
 *
 * hgt_gsample_layer_order, after each layer's last add_budget: from type_seq [B*2T] (device, the state's first-touch
 * numbers) member b's budget types in first-touch order go to type [T*B] (step k of the layer: type[k*B + b], -1 past
 * the member's last type) with step numbers step [T*B] = next_step[b] + k; next_step [B] advances by the member's type
 * count, and sel_off [T*(B+1)] holds, per step, the prefix sums over members of rooms [B*T] (region sizes) of the
 * selected types.  Run T select + add_budget steps with these; a member with type -1 does nothing in a step.
 *
 * hgt_gsample_graphed_layout, after the rebuild count pass: the write pass's node_off [B*T], blk_out [B*n_blocks],
 * self_off [B*T] and mem_out [B*4] that place every member in a padded signature layout, members joined type-major (as
 * merge_batches): member b's type-t rows start at row0[t] + (type-t nodes of members before b), its edges follow those of
 * the members before it, and edge_index is one [2, n_edges] array.  n_layer [B*T], type_seq [B*2T], totals [B*n_blocks]
 * from the state and the count pass.  grp_off [T+1] / grp_blk [n_blocks]: target type t's blocks in the order its edges
 * are laid out after its self loops.  blk_pair [n_blocks] / self_pair [T]: 0 when the block's (self loops') <source
 * type, relation> pair is in the signature, else a nonzero code; has_feat [T]: 1 when type t has a feature table;
 * type_cap [T]: the signature's rows of each type.  flags [8] (int32, device): [0..3] the sampler's, and the bounds this
 * call sets: [4] = 1 + the first type over type_cap, [5] = 1 when the edges exceed n_edges, [6] = the first pair code
 * met outside the signature, [7] = 1 + the first sampled type without a table.  With any flag set every table is -1 (the
 * write pass then writes nothing) and *n_real_edges (device) is 0; otherwise it is the edge count.
 *
 * hgt_gsample_graphed_rows: node_id[node_off + r] = the sampled id of ser r of every laid-out (member, type); the other
 * rows keep their value.  hgt_gsample_graphed_pad: edges n_real_edges.. n_edges - 1 become self loops on pad_node with
 * type 0 and time 120; with any of flags [8] set, all n_values of feature (float32, or bf16 when bf16 != 0) become NaN. */
int hgt_gsample_layer_order(const int64_t* type_seq, int32_t n_members, int32_t num_types, const int64_t* rooms,
                            int64_t* next_step, int32_t* type, int64_t* step, int64_t* sel_off, void* stream);
int hgt_gsample_graphed_layout(int32_t n_members, int32_t num_types, int32_t n_blocks, const int64_t* n_layer,
                               const int64_t* type_seq, const int64_t* totals, const int32_t* grp_off,
                               const int32_t* grp_blk, const int32_t* blk_pair, const int32_t* self_pair,
                               const int32_t* has_feat, const int64_t* row0, const int64_t* type_cap, int64_t n_edges,
                               int32_t* flags, int64_t* node_off, int64_t* blk_out, int64_t* self_off, int64_t* mem_out,
                               int64_t* n_real_edges, void* stream);
int hgt_gsample_graphed_rows(const hgt_gsample_hash_state* h_state, const int64_t* node_off, int64_t max_rows,
                             int64_t* node_id, void* stream);
int hgt_gsample_graphed_pad(const int64_t* n_real_edges, int64_t n_edges, int64_t pad_node, const int32_t* flags,
                            int64_t* edge_index, int64_t* edge_type, int64_t* edge_time, void* feature,
                            int64_t n_values, int32_t bf16, void* stream);

/* Disjoint union of B batches in the to_torch layout (sampler.py: merge_batches).  The member structs live in DEVICE
 * memory.  loc_off [B*(T+1)]: member b's first local row of each type (loc_off[b*(T+1)+T] = its node count); uoff [B*T]:
 * the union row of member b's first type-t row (type-major: node_type of the union is sorted).  member_rows [sum N_b]:
 * the union row of every member row, member b's at node_base.  Edges go to edge_base + e, endpoints remapped (ids
 * outside the member become -1).  node_feature may be NULL (then the members' are not read). */
typedef struct {
  const float* node_feature;
  const int64_t* edge_index;
  const int64_t* edge_type;
  const int64_t* edge_time;
  int64_t n_nodes, n_edges;
  int64_t node_base, edge_base;
} hgt_merge_member;
int hgt_merge_batches(const hgt_merge_member* members, int32_t n_members, int32_t num_types, const int64_t* loc_off,
                      const int64_t* uoff, int64_t max_rows, int64_t max_edges, int64_t n_edges, int32_t feat_dim,
                      int64_t* node_type, float* node_feature, int64_t* member_rows, int64_t* edge_index,
                      int64_t* edge_type, int64_t* edge_time, void* stream);
/* The same union of bf16 feature rows: the members' node_feature pointers and node_feature are bf16 [*, feat_dim]. */
int hgt_merge_batches_bf16(const hgt_merge_member* members, int32_t n_members, int32_t num_types, const int64_t* loc_off,
                           const int64_t* uoff, int64_t max_rows, int64_t max_edges, int64_t n_edges, int32_t feat_dim,
                           int64_t* node_type, void* node_feature, int64_t* member_rows, int64_t* edge_index,
                           int64_t* edge_type, int64_t* edge_time, void* stream);

/* Device-side build of one adjacency block from an edge array (sampler.py: DeviceGraph.from_edges).  Edge i, in array
 * order, sets d[tgt[i]][src[i]] = time[i] in a dict of dicts; the block is that dict in the CSR form of
 * hgt_gsample_block: rows in order of each target's first appearance, a row's neighbours in order of the pair's first
 * appearance, a repeated pair keeping its first place and its last time.  tgt / src / time [n_edges] are DEVICE int64
 * arrays (ids in [0, tgt_max] / [0, src_max]); time may be NULL (every time is None).  n_edges < 2^31.
 * hgt_ingest_block_sort sorts the edges in the workspace and writes stats [4] (DEVICE int64): the number of rows, the
 * number of entries (distinct pairs), and the least and greatest kept time (INT64_MAX / INT64_MIN when there is none or
 * time is NULL).  The caller reads them back, chooses the block's width and allocates its arrays; then
 * hgt_ingest_block_write, given the same tgt / src / time, the stats' counts and the same workspace (once per sort),
 * writes row_of [n_row_of] (>= tgt_max + 1 entries, -1 = no row), ptr [n_rows + 1], nbr and time_out [n_entries]: int32
 * arrays with INT32_MIN for a NULL time when narrow != 0 (HGT_BLOCK_NARROW), int64 with no_time otherwise.  Values are
 * not range-checked against the width.  workspace: hgt_ingest_workspace_bytes(n_edges), 48 bytes per edge + CUB scratch. */
int hgt_ingest_workspace_bytes(int64_t n_edges, size_t* out_bytes);
int hgt_ingest_block_sort(const int64_t* tgt, const int64_t* src, const int64_t* time, int64_t n_edges, int64_t tgt_max,
                          int64_t src_max, int64_t* stats, void* workspace, size_t workspace_bytes, void* stream);
int hgt_ingest_block_write(const int64_t* tgt, const int64_t* src, const int64_t* time, int64_t n_edges, int64_t n_rows,
                           int64_t n_entries, int32_t narrow, int64_t no_time, void* row_of, int64_t n_row_of, void* ptr,
                           void* nbr, void* time_out, void* workspace, size_t workspace_bytes, void* stream);

/* Node features derived from the sampler's blocks (sampler.py: mag_features, the ogbn-mag preprocessing rules).
 * `blocks` is a DEVICE array of n_blocks descriptors (the DeviceGraph's own, device- or host-placed, narrow or wide),
 * all with one target type of n_nodes ids; a block's row_of may be shorter than n_nodes (ids past it have no row).
 * hgt_feat_degree: deg[id] (DEVICE int64 [n_nodes]) = the sum over the blocks of id's row length, an integer sum, and
 * out[id * ld_out] = (float)log10((double)deg[id]), -inf for 0.
 * hgt_feat_neighbour_mean: for each id, the mean of the source rows src[s * src_ld + 0 .. feat_dim) over every entry s of
 * id's rows in the given blocks, in block order (a pair in two blocks counts twice), summed in fp64 in a fixed order
 * and divided by the entry count; zero for an id with no entries.  src is a DEVICE fp32 table, or fp64 when src_fp64,
 * and every neighbour id must be a row of it (not checked).  The mean is written as fp64 to out64 (row stride ld64)
 * and/or, rounded once, as fp32 to out32 (row stride ld32); either may be NULL, not both.  Both passes are bitwise
 * repeatable; nothing is allocated or synchronised. */
int hgt_feat_degree(const hgt_gsample_block* blocks, int32_t n_blocks, int64_t n_nodes, int64_t* deg, float* out,
                    int64_t ld_out, void* stream);
int hgt_feat_neighbour_mean(const hgt_gsample_block* blocks, int32_t n_blocks, int64_t n_nodes, const void* src,
                            int32_t src_fp64, int64_t src_ld, int32_t feat_dim, double* out64, int64_t ld64,
                            float* out32, int64_t ld32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HGT_B200_H */
