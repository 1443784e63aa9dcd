"""ctypes binding of libhgt_b200.so (C ABI declared in include/hgt_b200.h).

The library is built in-tree by ``pyhgt_b200/build.py`` (nvcc, sm_90a).  There is NO fallback: if the
shared object is missing or a symbol is absent, loading raises.
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libhgt_b200.so")

_c = ctypes
_p = _c.c_void_p
_i32 = _c.c_int32
_i64 = _c.c_int64
_sz = _c.c_size_t
_f32 = _c.c_float

# name -> argtypes; every function returns int except where noted.  Mirrors include/hgt_b200.h.
SIGNATURES = {
    "hgt_abi_version": [],
    "hgt_plan_workspace_bytes": [_i64, _i64, _c.POINTER(_sz)],
    "hgt_plan_nodes": [_p, _i64, _i32, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_plan_edges_sort": [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_plan_edges_fill": [_p, _p, _p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _p, _p, _i32, _i32, _p, _p, _p, _p],
    "hgt_plan_tiles": [_p, _i64, _i64, _i32, _i32, _p, _i64, _p, _i64, _p, _c.POINTER(_i32), _p, _sz, _p],
    "hgt_gather_rows": [_p, _p, _i64, _i32, _p, _p],
    "hgt_halo_pull": [_c.c_uint64, _p, _p, _i64, _i32, _i64, _p, _p],
    "hgt_halo_pull_split": [_c.c_uint64, _p, _p, _p, _i64, _i32, _i32, _i64, _p, _p, _p, _p],
    "hgt_halo_push_split": [_p, _p, _p, _p, _i64, _i32, _i32, _i64, _c.c_uint64, _c.c_uint64, _p, _p],
    "hgt_fold_weights": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p,
                         _p, _p, _p],
    "hgt_concat_linears": [_p, _p, _i32, _i32, _i32, _p, _p, _p],
    "hgt_typed_linear_workspace_bytes": [_p, _i32, _i32, _i32, _i32, _c.POINTER(_sz)],
    "hgt_typed_linear": [_p, _i64, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i32, _p, _sz, _p],
    "hgt_edge_workspace_bytes": [_i32, _i32, _i32, _c.POINTER(_sz)],
    "hgt_edge_forward": [_p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i64, _i32, _i32, _i32, _p, _p,
                         _p, _p, _p, _p, _sz, _i32, _p, _p, _i32, _p, _p],
    "hgt_typed_linear_presplit_workspace_bytes": [_p, _i32, _i32, _i32, _c.POINTER(_sz)],
    "hgt_typed_linear_presplit": [_p, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _p, _sz, _p],
    "hgt_edge_backward": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _i32, _i32, _i64, _i64, _p, _p, _p, _p, _sz,
                          _p, _p],
    "hgt_typed_linear_bwd_workspace_bytes": [_p, _i32, _p, _i32, _i32, _i64, _i64, _i32, _i32, _i32, _c.POINTER(_sz)],
    "hgt_typed_linear_bwd": [_p, _p, _p, _i64, _p, _i64, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i32, _p, _p, _p,
                             _i32, _p, _sz, _p],
    "hgt_act_split": [_p, _i64, _i64, _i32, _i32, _p, _p, _p, _p],
    "hgt_update_backward": [_p, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p, _p, _p],
    "hgt_fold_backward": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _p, _p,
                          _p, _p, _p, _p, _p],
    "hgt_conv_workspace_bytes": [_p, _c.POINTER(_sz)],
    "hgt_conv_forward": [_p, _p, _sz, _p],
    "hgt_update_epilogue": [_p, _p, _p, _i32, _p, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p],
    # inference over each type's destination extent (plan.GraphPlan.dst_extent)
    "hgt_plan_dst_end": [_p, _p, _p, _i64, _i32, _p, _p],
    "hgt_update_epilogue_dst": [_p, _p, _p, _i32, _p, _p, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p],
    # deterministic training backward (torch.use_deterministic_algorithms)
    "hgt_plan_source_index": [_p, _p, _p, _i64, _i64, _i32, _p, _p, _p, _p, _sz, _p],
    "hgt_plan_source_index_pos": [_p, _p, _p, _i64, _i64, _i32, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_edge_backward_det_workspace_bytes": [_i32, _i32, _i32, _c.POINTER(_sz)],
    "hgt_edge_backward_dst": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i32, _i32, _p, _p, _p,
                              _sz, _p, _p],
    "hgt_edge_backward_rows": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _p, _i32, _i32, _p, _i32, _i32, _i32, _p,
                               _p, _sz, _p, _p],
    "hgt_typed_linear_bwd_det_workspace_bytes": [_p, _i32, _p, _i32, _i32, _i64, _i64, _i32, _i32, _i32,
                                                 _c.POINTER(_sz)],
    "hgt_typed_linear_bwd_det": [_p, _p, _p, _i64, _p, _i64, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i32, _p, _p,
                                 _p, _i32, _p, _sz, _p],
    "hgt_update_backward_det_workspace_bytes": [_i64, _i32, _i32, _c.POINTER(_sz)],
    "hgt_update_backward_det": [_p, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_fold_backward_det": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _p,
                              _p, _p, _p, _p, _p, _p],
    # bf16 gather tables (HGT layers under torch.autocast(dtype=torch.bfloat16)): same arguments as the fp32 twins
    "hgt_typed_linear_bf16": [_p, _i64, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i32, _p, _sz, _p],
    "hgt_typed_linear_presplit_bf16": [_p, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _p, _sz, _p],
    # 24-bit gather tables: the fp32 twins' arguments with (out, t24_off, out24) for out
    "hgt_typed_linear_t24": [_p, _i64, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i64, _p, _i32, _p, _sz, _p],
    "hgt_typed_linear_presplit_t24": [_p, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i64, _p, _p, _sz, _p],
    # bs16 gather tables: the 24-bit calls' arguments
    "hgt_gather_table_format": [_i32, _i64, _i64, _c.POINTER(_i32)],
    "hgt_gather_table_row_bytes": [_i32, _i64, _c.POINTER(_i64)],
    "hgt_typed_linear_bs16": [_p, _i64, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i64, _p, _i32, _p, _sz, _p],
    "hgt_typed_linear_presplit_bs16": [_p, _p, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i64, _p, _p, _sz, _p],
    "hgt_edge_forward_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i64, _i32, _i32, _i32, _p, _p,
                              _p, _p, _p, _p, _sz, _i32, _p, _p, _i32, _p, _p],
    # 24-bit gather tables (inference forwards that keep nothing for a backward): same arguments as the bf16 twins
    "hgt_edge_forward_t24": [_p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i64, _i32, _i32, _i32, _p, _p,
                             _p, _p, _p, _p, _sz, _i32, _p, _p, _i32, _p, _p],
    "hgt_edge_forward_bs16": [_p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i64, _i32, _i32, _i32, _p, _p,
                              _p, _p, _p, _p, _sz, _i32, _p, _p, _i32, _p, _p],
    "hgt_edge_backward_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _i32, _i32, _i64, _i64, _p, _p, _p, _p,
                               _sz, _p, _p],
    "hgt_edge_backward_dst_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i32, _i32, _p, _p,
                                   _p, _sz, _p, _p],
    "hgt_edge_backward_rows_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _p, _i32, _i32, _p, _i32, _i32, _i32,
                                    _p, _p, _sz, _p, _p],
    # gradient of att (a loss term reads HGTConv.att): C / CSR-order datt, then the edge backward passes with datt
    "hgt_edge_att_grad_workspace_bytes": [_i32, _i32, _c.POINTER(_sz)],
    "hgt_edge_att_grad_prep": [_p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i32, _p, _p, _p, _sz, _p, _p],
    "hgt_edge_backward_att": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _i32, _i32, _i64, _i64, _p, _p,
                              _p, _p, _sz, _p, _p],
    "hgt_edge_backward_dst_att": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i32, _i32,
                                  _p, _p, _p, _sz, _p, _p],
    "hgt_edge_backward_rows_att": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _p, _i32, _i32, _p, _i32, _i32,
                                   _i32, _p, _p, _sz, _p, _p],
    "hgt_edge_backward_att_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _i32, _i32, _i64, _i64, _p,
                                   _p, _p, _p, _sz, _p, _p],
    "hgt_edge_backward_dst_att_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i64, _i32,
                                       _i32, _p, _p, _p, _sz, _p, _p],
    "hgt_edge_backward_rows_att_bf16": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _i64, _p, _i32, _i32, _p, _i32,
                                        _i32, _i32, _p, _p, _sz, _p, _p],
    # HGSampling on the GPU, B subgraphs per pass (sampler.sample_subgraphs_cuda), and their union (merge_batches)
    "hgt_gsample_batch_add_budget_workspace_bytes": [_i32, _i64, _i32, _i64, _c.POINTER(_sz)],
    "hgt_gsample_batch_add_budget": [_p, _p, _p, _i32, _p, _p, _p, _p, _i64, _p, _i64, _i32, _i64, _i64, _p, _p, _sz,
                                     _p],
    "hgt_gsample_batch_select_workspace_bytes": [_i32, _i64, _c.POINTER(_sz)],
    "hgt_gsample_batch_select": [_p, _p, _p, _p, _i64, _i64, _i64, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_gsample_rebuild_workspace_bytes": [_i64, _c.POINTER(_sz)],
    "hgt_gsample_batch_rebuild_count": [_p, _p, _i32, _p, _p, _i64, _i64, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_gsample_batch_rebuild_write": [_p, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _i64, _p, _i32, _p, _p, _p,
                                        _p, _p, _p, _p],
    # graphs in page-locked host memory (sampler.DeviceGraph(..., placement="host"))
    "hgt_host_register": [_p, _sz, _c.POINTER(_p)],
    "hgt_host_unregister": [_p],
    # bf16 feature tables of the device sampler (DeviceGraph(..., feature_dtype=torch.bfloat16))
    "hgt_gsample_gather_features_bf16": [_p, _i32, _p, _p, _i64, _p, _p],
    "hgt_gsample_batch_rebuild_count_host": [_p, _p, _i32, _p, _p, _i64, _i64, _p, _p, _i64, _p, _p, _p, _p, _p, _sz,
                                             _p],
    "hgt_gsample_batch_rebuild_write_host": [_p, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p,
                                             _i32, _p, _p, _p, _p, _p, _p, _p],
    # the hashed sampler state, sized by the sample (sample_subgraphs_cuda on graphs with large id ranges)
    "hgt_gsample_hash_insert_seeds": [_p, _i64, _p, _p, _p, _p, _p, _p],
    "hgt_gsample_hash_add_budget": [_p, _p, _p, _i32, _p, _p, _p, _p, _i64, _p, _i64, _i32, _i64, _i64, _p, _p, _sz,
                                    _p],
    "hgt_gsample_hash_select_workspace_bytes": [_i32, _i64, _c.POINTER(_sz)],
    "hgt_gsample_hash_select": [_p, _p, _p, _p, _i64, _i64, _i64, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_gsample_hash_rebuild_count": [_p, _p, _i32, _p, _p, _i64, _i64, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_gsample_hash_rebuild_write": [_p, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _i64, _p, _i32, _p, _p, _p,
                                       _p, _p, _p, _p],
    "hgt_gsample_hash_rebuild_count_host": [_p, _p, _i32, _p, _p, _i64, _i64, _p, _p, _i64, _p, _p, _p, _p, _p, _sz,
                                            _p],
    "hgt_gsample_hash_rebuild_write_host": [_p, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _i64, _p, _i64, _p,
                                            _i32, _p, _p, _p, _p, _p, _p, _p],
    "hgt_merge_batches": [_p, _i32, _i32, _p, _p, _i64, _i64, _i64, _i32, _p, _p, _p, _p, _p, _p, _p],
    # bf16 node features end to end (sample_subgraph(s)_cuda(..., feature_dtype=torch.bfloat16), GNN's adapter)
    "hgt_gsample_gather_rows_bf16": [_p, _i32, _p, _p, _i64, _p, _p],
    "hgt_merge_batches_bf16": [_p, _i32, _i32, _p, _p, _i64, _i64, _i64, _i32, _p, _p, _p, _p, _p, _p, _p],
    "hgt_typed_linear_bf16a": [_p, _i64, _p, _p, _i32, _i32, _p, _p, _i32, _p, _p, _i32, _p, _sz, _p],
    "hgt_typed_linear_bwd_bf16a": [_p, _i64, _p, _i64, _i32, _i32, _p, _p, _i32, _p, _p, _p, _i32, _p, _sz, _p],
    "hgt_typed_linear_bwd_bf16a_det": [_p, _i64, _p, _i64, _i32, _i32, _p, _p, _i32, _p, _p, _p, _i32, _p, _sz, _p],
    # the sampler's graph built on the device from typed edge arrays (sampler.DeviceGraph.from_edges)
    "hgt_ingest_workspace_bytes": [_i64, _c.POINTER(_sz)],
    "hgt_ingest_block_sort": [_p, _p, _p, _i64, _i64, _i64, _p, _p, _sz, _p],
    "hgt_ingest_block_write": [_p, _p, _p, _i64, _i64, _i64, _i32, _i64, _p, _i64, _p, _p, _p, _p, _sz, _p],
    # ogbn-mag node features from the sampler's blocks (sampler.mag_features)
    "hgt_feat_degree": [_p, _i32, _i64, _p, _p, _i64, _p],
    "hgt_feat_neighbour_mean": [_p, _i32, _i64, _p, _i32, _i64, _i32, _p, _i64, _p, _i64, _p],
    # sampling with fixed shapes and no read-back (sampler.GraphedSampler)
    "hgt_gsample_layer_order": [_p, _i32, _i32, _p, _p, _p, _p, _p, _p],
    "hgt_gsample_graphed_layout": [_i32, _i32, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p,
                                   _p, _p],
    "hgt_gsample_graphed_rows": [_p, _p, _i64, _p, _p],
    "hgt_gsample_graphed_pad": [_p, _i64, _i64, _p, _p, _p, _p, _p, _i64, _i32, _p],
    # trimmed forward (GNN.forward(out_nodes=), trim.py)
    "hgt_trim_layout": [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p],
    "hgt_trim_layout_bounded": [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _i64, _i32, _p, _i64, _p, _p, _p, _p, _p,
                                _p, _p, _p, _sz, _p],
    "hgt_plan_range_tiles": [_p, _i64, _i64, _p, _i32, _i64, _i32, _i32, _p, _i64, _p, _i64, _p, _p, _sz, _p],
    "hgt_plan_mask_rows": [_p, _p, _p, _i32, _i64, _i32, _p, _p],
    # fused dropout (HGTConv.fused_dropout / GNN.fused_dropout): the plain twins' arguments + (seed, p) before the stream
    "hgt_update_epilogue_drop": [_p, _p, _p, _i32, _p, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p, _f32, _p],
    "hgt_update_backward_drop": [_p, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p, _p, _p, _f32, _p],
    "hgt_update_backward_drop_det": [_p, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p, _p, _p, _sz, _p,
                                     _f32, _p],
    "hgt_tanh_dropout": [_p, _i64, _i64, _i32, _p, _f32, _p, _p],
    "hgt_tanh_dropout_bwd": [_p, _p, _i64, _i64, _i32, _p, _f32, _p, _p],
}

class ConvArgs(ctypes.Structure):
    """Mirror of `hgt_conv_args` (include/hgt_b200.h); field order and types must match the C struct exactly
    (checked against hgt_conv_args_size() in tests/test_capi.py)."""
    _I64 = ["n_nodes", "n_edges", "kv_rows", "cat_rows", "q_off", "kv_off", "proj_elems"]
    _I32 = ["num_types", "num_relations", "n_heads", "d_in", "d_out", "n_pairs", "use_rte", "use_norm", "edge_variant",
            "linear_impl", "n_tiles", "n_split", "n_hubs", "n_proj_groups", "n_rte_groups", "n_upd_groups"]
    _PTR = ["perm", "type_row0", "type_active", "out_map", "row_ptr", "kv_row", "rte_row", "csr_eid", "tiles", "hubs",
            "d_tile_counts", "pair_type", "pair_rel", "cat_row0", "q_row0",
            "proj_groups", "h_proj_groups", "proj_cblocks", "rte_groups", "h_rte_groups", "rte_cblocks",
            "rt_groups", "h_rt_groups", "rt_cblocks", "upd_groups", "h_upd_groups", "upd_cblocks",
            "wq", "bq", "wk", "bk", "wv", "bv", "wa", "ba", "norm_w", "norm_b",
            "relation_att", "relation_msg", "relation_pri", "skip", "emb_weight", "emb_lin_w", "emb_lin_b",
            "x", "x_hi", "x_lo", "out", "att", "out_hi", "out_lo", "type_dst"]
    _fields_ = ([(n, ctypes.c_int64) for n in _I64] + [(n, ctypes.c_int32) for n in _I32] +
                [(n, ctypes.c_void_p) for n in _PTR])


LIN_GROUP_DTYPE = np.dtype([("a_row0", "<i8"), ("m", "<i8"), ("w_row0", "<i4"), ("n_cblocks", "<i4"),
                            ("cb_first", "<i4"), ("has_bias", "<i4")])
LIN_CBLOCK_DTYPE = np.dtype([("out_off", "<i8"), ("ld", "<i8")])
assert LIN_GROUP_DTYPE.itemsize == 32 and LIN_CBLOCK_DTYPE.itemsize == 16

_lib = None


class HgtError(RuntimeError):
    pass


def load():
    """Load the shared library once and attach argtypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise HgtError("libhgt_b200.so not found at %s — run `python -m pyhgt_b200.build` "
                       "(or __graft_entry__.build()); there is no CPU fallback" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.hgt_last_error.restype = _c.c_char_p
    lib.hgt_last_error.argtypes = []
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing: loud by design
        fn.restype = _c.c_int
        fn.argtypes = args
    lib.hgt_kernel_launches.restype = _c.c_uint64
    lib.hgt_kernel_launches.argtypes = []
    lib.hgt_conv_args_size.restype = _c.c_uint64
    lib.hgt_conv_args_size.argtypes = []
    lib.hgt_sampler_budget_update.restype = _c.c_int64       # host helper of sampler.py: returns a count, not a status
    lib.hgt_sampler_budget_update.argtypes = [_p, _p, _i64, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p, _p, _p]
    lib.hgt_sampler_add_budget.restype = _c.c_int64
    lib.hgt_sampler_add_budget.argtypes = [_p, _p, _i64, _p, _c.c_int32, _p, _c.c_int32, _i64, _p, _p, _i64, _i64, _p]
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().hgt_last_error()
        raise HgtError("%s failed (code %d): %s" % (what, rc, msg.decode() if msg else "?"))


def call(name, *args):
    lib = load()
    check(getattr(lib, name)(*args), name)


TABLE_F32, TABLE_T24, TABLE_BS16 = 0, 1, 2                     # HGT_TABLE_* (include/hgt_b200.h)
TABLE_SUFFIX = {TABLE_F32: "", TABLE_T24: "_t24", TABLE_BS16: "_bs16"}   # entry-point suffix of a format


def gather_table_format(d, table_rows, device):
    """hgt_gather_table_format for an inference forward's [K'|V'] table of table_rows rows on `device`."""
    import torch
    out = _c.c_int32()
    call("hgt_gather_table_format", d, table_rows, torch.cuda.get_device_properties(device).L2_cache_size,
         _c.byref(out))
    return out.value


def gather_table_row_bytes(fmt, n):
    out = _c.c_int64()
    call("hgt_gather_table_row_bytes", fmt, n, _c.byref(out))
    return out.value


def kernel_launches():
    return int(load().hgt_kernel_launches())


def ptr(t):
    """Device (or host) address of a torch tensor, or None."""
    return None if t is None else t.data_ptr()
