"""Hop layout of a trimmed GNN forward, ``GNN.forward(..., out_nodes=)``: every layer computed only where the requested
output rows depend on it (PyG's ``trim_to_layer``, DGL's per-layer blocks).

``dist(v)`` is the length of the shortest path along edges (source -> destination) from v to any node of ``out_nodes``.
Layer l of L (1-based) must produce rows exactly for dist <= L - l, reads K'/V' rows of sources with dist <= L - l + 1,
and the input adapter is needed for dist <= L: a layer's output at v depends only on its input at v (skip connection,
LayerNorm) and at v's in-neighbours, whose dist is at most dist(v) + 1.

The layout reorders the batch so that every one of these sets is a prefix of each node type:

  * hgt_trim_layout (one pass on the device): the BFS distances, the nodes stably sorted by (type, min(dist, L+1)) —
    unknown types last, as in the plan's rank order — the batch's tensors in that order, and a [T, L+2] table of
    per-(type, hop) counts.  That table (with the range flags and the <source type, relation> presence) is the one
    device -> host read-back; the reordered batch is type-sorted with the original type counts and pairs, so its plan is
    the sync-free ``plan.build_plan(..., host_meta)``.
  * per layer a ``LayerView``: the hop plan with edge tiles over the layer's destination ranges only
    (hgt_plan_range_tiles), its active prefix per type (Q, a_linear, update) and its K'/V' row ranges (``kv_runs``).
    The deterministic backward's source index of a view holds only the edges of those destinations
    (plan.source_index, hgt_plan_mask_rows).

Rows a stage does not compute are zero: the adapter's and every layer's rows outside their prefix (see
autograd._UpdateEpilogue and conv.HGTConv._forward_impl), so no consumer can read an unwritten row.

Layouts are cached by the identity and version of (node_type, edge_index, edge_type, edge_time, out_nodes) and the
layer count, like plan.get_plan: a second forward or backward on the same batch synchronises nothing.
"""
import ctypes
import dataclasses
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import plan as _plan

_CACHE = []
_CACHE_SIZE = 4


@dataclass
class LayerView:
    plan: _plan.GraphPlan         # the hop plan with this layer's destination tiles
    active: tuple                 # [T] leading rows of each type the layer computes (dist <= L - l)
    kv_runs: tuple                # per pair, the K'/V' rows its edges read (dist <= L - l + 1): plan.layer_tables


@dataclass
class TrimLayout:
    n_layers: int
    counts: np.ndarray            # [T, L+2] nodes per (type, min(dist, L+1))
    dist: torch.Tensor            # [N] int32, original node order
    perm: torch.Tensor            # [N] int64: hop row -> original node
    out_rows: torch.Tensor        # [n_out] int64: hop row of every out_nodes entry
    plan: _plan.GraphPlan         # plan of the reordered (type-sorted) batch
    layers: list                  # [L] LayerView
    adapter_rows: tuple           # [T] leading rows of each type the input adapter computes (dist <= L)


def clear_trim_cache():
    _CACHE.clear()


def get_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers):
    tensors = (node_type, edge_index, edge_type, edge_time, out_nodes)
    extra = (int(num_types), int(num_relations), int(n_layers))
    hit = _plan._cache_lookup(tensors, extra, _CACHE)
    if hit is not None:
        return hit
    lay = build_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers)
    _plan._cache_store(tensors, extra, lay, _CACHE, _CACHE_SIZE)
    return lay


def build_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers):
    dev = node_type.device
    if dev.type != "cuda" or out_nodes.device != dev:
        raise _lib.HgtError("pyhgt_b200 runs on CUDA tensors only (node_type on %s, out_nodes on %s); there is no CPU "
                            "fallback" % (dev, out_nodes.device))
    nt = _plan._as_i64(node_type, "node_type", dev)
    ei = _plan._as_i64(edge_index, "edge_index", dev)
    et = _plan._as_i64(edge_type, "edge_type", dev)
    tm = _plan._as_i64(edge_time, "edge_time", dev)
    on = _plan._as_i64(out_nodes, "out_nodes", dev)
    if on.dim() != 1:
        raise ValueError("out_nodes must be a 1-D tensor of node ids, got shape %s" % (tuple(on.shape),))
    N = nt.numel()
    if ei.dim() != 2 or ei.shape[0] != 2:
        raise ValueError("edge_index must have shape [2, E], got %s" % (tuple(ei.shape),))
    E = ei.shape[1]
    if et.numel() != E or (tm is not None and tm.numel() != E):
        raise ValueError("edge_type / edge_time must have one entry per edge (E=%d)" % E)
    if N >= 2 ** 31 - 1024 or E >= 2 ** 31 - 1024:
        raise ValueError("graph too large for int32 CSR indices (N=%d, E=%d)" % (N, E))
    T, R, L = int(num_types), int(num_relations), int(n_layers)
    n_out = on.numel()
    st = _plan._stream()
    i32 = dict(dtype=torch.int32, device=dev)
    i64 = dict(dtype=torch.int64, device=dev)

    ws_bytes = ctypes.c_size_t()
    _lib.call("hgt_plan_workspace_bytes", N, E, ctypes.byref(ws_bytes))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    dist = torch.empty(max(N, 1), **i32)
    hop_perm = torch.empty(max(N, 1), **i32)
    hop_rank = torch.empty(max(N, 1), **i32)
    hop_nt = torch.empty(N, **i64)
    hop_ei = torch.empty((2, E), **i64)
    out_rows = torch.empty(n_out, **i64)
    n_counts = T * (L + 2)
    meta = torch.empty(n_counts + T * R + 4, **i32)
    _lib.call("hgt_trim_layout", ei.data_ptr(), et.data_ptr(), _lib.ptr(tm), nt.data_ptr(), N, E, T, R, on.data_ptr(),
              n_out, L, dist.data_ptr(), hop_perm.data_ptr(), hop_rank.data_ptr(), hop_nt.data_ptr(), hop_ei.data_ptr(),
              out_rows.data_ptr(), meta.data_ptr(), ws.data_ptr(), ws.numel(), st)
    meta_h = meta.cpu().numpy()                              # the one host read-back of a trimmed forward
    flags = meta_h[n_counts + T * R:]
    if flags[0]:
        raise IndexError("edge_index contains node ids outside [0, %d)" % N)
    if flags[1]:
        raise IndexError("edge_time contains values outside [0, %d) (RelTemporalEncoding table size)"
                         % _plan.RTE_MAX_LEN)
    if flags[2]:
        raise IndexError("out_nodes contains node ids outside [0, %d)" % N)
    counts = meta_h[:n_counts].reshape(T, L + 2).astype(np.int64)
    presence = meta_h[n_counts:n_counts + T * R].reshape(T, R)
    type_count = [int(c) for c in counts.sum(1)] + [N - int(counts.sum())]
    pairs = [(s, r) for s in range(T) for r in range(R) if presence[s, r]]
    hop = _plan.build_plan(hop_nt, hop_ei, et, tm, T, R, {"type_count": type_count, "sorted": True, "pairs": pairs})

    cum = np.cumsum(counts, 1)                               # cum[t, b]: nodes of type t with dist <= b
    layers = []
    for l in range(1, L + 1):
        active = tuple(int(cum[t, L - l]) for t in range(T))
        kv = [int(cum[t, L - l + 1]) for t in range(T)]
        kv_runs = tuple(((s, r), ((0, kv[s]),)) for (s, r) in hop.pairs)
        ranges = [(hop.type_row0[t], hop.type_row0[t] + active[t]) for t in range(T) if active[t] > 0]
        layers.append(LayerView(plan=_range_view(hop, ranges), active=active, kv_runs=kv_runs))
    return TrimLayout(n_layers=L, counts=counts, dist=dist[:N], perm=hop_perm[:N].long(), out_rows=out_rows, plan=hop,
                      layers=layers, adapter_rows=tuple(int(cum[t, L]) for t in range(T)))


def _range_view(plan, ranges):
    """`plan` with edge tiles over the destination row ranges only (hgt_plan_range_tiles, sync-free) and its own
    layer-table and source-index caches."""
    dev = plan.row_ptr.device
    i32 = dict(dtype=torch.int32, device=dev)
    N, E = plan.n_nodes, plan.n_edges
    n_rows = sum(b - a for a, b in ranges)
    rng = _plan._to_dev_async(np.asarray(ranges if ranges else [(0, 0)], dtype=np.int32).reshape(-1), dev)
    split = _plan.TILE_SPLIT_EDGES
    max_tiles = (2 * E + N) // (2 * _plan.TILE_TARGET_EDGES) + 3 * (E // split) + 16 + len(ranges)
    max_hubs = E // split + 1
    tiles = torch.empty((max_tiles, 4), **i32)
    hubs = torch.empty((max_hubs, 4), **i32)
    counts = torch.zeros(4, **i32)
    ws_bytes = ctypes.c_size_t()
    _lib.call("hgt_plan_workspace_bytes", N, E, ctypes.byref(ws_bytes))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    _lib.call("hgt_plan_range_tiles", plan.row_ptr.data_ptr(), N, E, rng.data_ptr(), len(ranges), n_rows,
              _plan.TILE_TARGET_EDGES, split, tiles.data_ptr(), max_tiles, hubs.data_ptr(), max_hubs,
              counts.data_ptr(), ws.data_ptr(), ws.numel(), _plan._stream())
    has_hub = E > split
    return dataclasses.replace(plan, tiles=tiles, n_tiles=max_tiles if n_rows > 0 else 0,
                               n_split=2 * (E // split) + 1 if has_hub else 0, hubs=hubs,
                               n_hubs=max_hubs if has_hub else 0, tile_counts_dev=counts, dst_ranges=rng,
                               n_dst_ranges=len(ranges), _layer_tables={}, _source_index={})
