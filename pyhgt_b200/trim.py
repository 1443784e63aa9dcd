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
  * with a ``TrimSignature`` (hop bounds known on the host) hgt_trim_layout_bounded places the same order into slot
    regions of the bounds' sizes instead, padded with inert rows, and nothing is read back: the layout of a new batch is
    sync-free and a CUDA graph can capture it (graphed.py).  The <source type, relation> pairs then come from the batch's
    cached plan.  Overflow (a class larger than its bound) and out-of-range ids are left in device flags: the trimmed
    forward writes NaN into its rows, and ``TrimLayout.check()`` raises.
  * per layer a ``LayerView``: the hop plan with edge tiles over the layer's destination ranges only
    (hgt_plan_range_tiles), its active prefix per type (Q, a_linear, update) and its K'/V' row ranges (``kv_runs``).
    The deterministic backward's source index of a view holds only the edges of those destinations
    (plan.source_index, hgt_plan_mask_rows).

Everything derived from the layout on the host (prefixes, K'/V' runs, row ranges, adapter rows, the hop plan's type
counts) is computed from the per-(type, hop) slot sizes: the counts read back, or the signature's bounds.

Rows a stage does not compute are zero: the adapter's and every layer's rows outside their prefix (see
autograd._UpdateEpilogue and conv.HGTConv._forward_impl), so no consumer can read an unwritten row.

Layouts are cached by the identity and version of (node_type, edge_index, edge_type, edge_time, out_nodes), the layer
count and the signature, like plan.get_plan: a second forward or backward on the same batch synchronises nothing.  While
a CUDA graph is being captured the cache is bypassed, so the captured layout kernels lay out every replayed batch.
"""
import contextlib
import ctypes
import dataclasses
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import plan as _plan

_CACHE = []
_CACHE_SIZE = 4


class TrimSignature:
    """Host-known slot sizes of the hop layout of a family of batches: ``hop_bounds[t][b]`` rows for the nodes of type t
    at hop distance b (b = L+1: farther).  Hop class L+1 is never computed or read, so its nodes may be left out (bound
    0, as ``for_batches`` sizes it); any other class larger than its bound is an overflow (NaN rows, ``check()`` raises)."""

    def __init__(self, hop_bounds, n_layers):
        L = int(n_layers)
        b = np.array(hop_bounds, dtype=np.int64)
        if L < 1 or b.ndim != 2 or b.shape[0] < 1 or b.shape[1] != L + 2:
            raise ValueError("hop_bounds must be a [num_types, n_layers + 2] table, got shape %s for n_layers=%d"
                             % (b.shape, L))
        if (b < 0).any():
            raise ValueError("hop_bounds must be non-negative")
        if b.sum() + 1 >= 2 ** 31 - 1024:
            raise ValueError("hop_bounds sum past the int32 row range")
        self.hop_bounds = b
        self.hop_bounds.setflags(write=False)
        self.n_layers = L
        self.num_types = b.shape[0]
        self.n_rows = int(b.sum()) + 1                     # + the pad row (out-of-range type) that dropped nodes map to

    def key(self):
        return (self.n_layers, self.hop_bounds.shape, self.hop_bounds.tobytes())

    @classmethod
    def for_batches(cls, batches, out_nodes_list, n_layers, slack=0.0, *, num_types, num_relations):
        """Bounds covering every (batch, out_nodes) pair: the per-(type, hop) maximum of their counts times (1 + slack),
        rounded up, with hop class L+1 left out.  `batches`: tuples that start (node_feature, node_type, edge_time,
        edge_index, edge_type), as sample_subgraphs_cuda returns them.  One device -> host read-back for all of them."""
        batches, outs = list(batches), list(out_nodes_list)
        if len(batches) != len(outs) or not batches:
            raise ValueError("for_batches needs one out_nodes tensor per batch (got %d batches, %d out_nodes)"
                             % (len(batches), len(outs)))
        if not slack >= 0:
            raise ValueError("slack must be >= 0, got %r" % (slack,))
        T, R, L = int(num_types), int(num_relations), int(n_layers)
        metas = []
        for b, on in zip(batches, outs):
            args = _check_args(b[1], b[3], b[4], b[2], on)
            metas.append(_launch(*args, T, R, L)[-1][:T * (L + 2) + T * R + 4])
        meta = torch.stack(metas).cpu().numpy()             # the one read-back
        for m, b in zip(meta, batches):
            _raise_flags(m[T * (L + 2) + T * R:], int(b[1].numel()))
        counts = meta[:, :T * (L + 2)].reshape(-1, T, L + 2).max(0).astype(np.float64)
        bounds = np.ceil(counts * (1.0 + float(slack))).astype(np.int64)
        bounds[:, L + 1] = 0
        return cls(bounds, L)


@dataclass
class LayerView:
    plan: _plan.GraphPlan         # the hop plan with this layer's destination tiles
    active: tuple                 # [T] leading rows of each type the layer computes (dist <= L - l)
    kv_runs: tuple                # per pair, the K'/V' rows its edges read (dist <= L - l + 1): plan.layer_tables


@dataclass
class TrimLayout:
    n_layers: int
    counts: np.ndarray            # [T, L+2] nodes per (type, min(dist, L+1)); None for a signature layout (on the device)
    dist: torch.Tensor            # [N] int32, original node order
    perm: torch.Tensor            # [rows] int64: hop row -> original node (N on a padding row)
    out_rows: torch.Tensor        # [n_out] int64: hop row of every out_nodes entry
    plan: _plan.GraphPlan         # plan of the reordered (type-sorted) batch
    layers: list                  # [L] LayerView
    adapter_rows: tuple           # [T] leading rows of each type the input adapter computes (dist <= L)
    bounds: np.ndarray = None     # [T, L+2] slot rows per (type, hop): the counts, or the signature's bounds
    counts_dev: torch.Tensor = None   # [T, L+2] int32 actual counts, on the device
    flags_dev: torch.Tensor = None    # signature layouts: [4] int32 device flags (edge ids, edge_time, out_nodes, overflow)
    bad: torch.Tensor = None          # signature layouts: 0-dim device bool, any flag set (the forward's rows become NaN)
    gather: torch.Tensor = None       # signature layouts: perm with padding rows pointing at node 0 (int64) ...
    pad_rows: torch.Tensor = None     # ... and [rows, 1] bool, true on padding rows: the gather's rows to zero

    @property
    def padded(self):
        return self.flags_dev is not None

    def check(self):
        """Signature layouts leave their errors on the device: read the flags back (one host sync) and raise as the
        read-back build does, ValueError for an overflow."""
        if self.flags_dev is None:
            return
        f = self.flags_dev.cpu().numpy()
        _raise_flags(f, self.dist.numel())
        if f[3]:
            raise ValueError("a (type, hop) class of this batch has more nodes than its TrimSignature bound (the "
                             "trimmed forward's rows are NaN); actual counts per (type, hop): %s"
                             % self.counts_dev.cpu().numpy().tolist())


def clear_trim_cache():
    _CACHE.clear()


@contextlib.contextmanager
def _sync_forbidden():
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(prev)


def get_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers,
               signature=None, pairs=None):
    """`signature` (optional): a TrimSignature; the layout is then built without any synchronisation (enforced with
    torch.cuda.set_sync_debug_mode("error")) from the bounds and `pairs`, the batch's <source type, relation> pairs."""
    tensors = (node_type, edge_index, edge_type, edge_time, out_nodes)
    extra = (int(num_types), int(num_relations), int(n_layers), None if signature is None else signature.key())
    capturing = torch.cuda.is_current_stream_capturing()
    if not capturing:
        hit = _plan._cache_lookup(tensors, extra, _CACHE)
        if hit is not None:
            return hit
    if signature is None:
        lay = build_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers)
    else:
        with _sync_forbidden():
            lay = build_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations,
                               n_layers, signature, pairs)
    if not capturing:
        _plan._cache_store(tensors, extra, lay, _CACHE, _CACHE_SIZE)
    return lay


def _check_args(node_type, edge_index, edge_type, edge_time, out_nodes):
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
    return nt, ei, et, tm, on


def _launch(nt, ei, et, tm, on, T, R, L, bounds=None):
    """hgt_trim_layout (bounds None: exact, one row per node) or hgt_trim_layout_bounded (host [T, L+2] bounds plus the
    pad row).  Returns (dist, hop_perm, hop_nt, hop_ei, out_rows, meta), all on the device."""
    dev = nt.device
    N, E, n_out = nt.numel(), ei.shape[1], on.numel()
    n_rows = N if bounds is None else int(bounds.sum()) + 1
    st = _plan._stream()
    i32 = dict(dtype=torch.int32, device=dev)
    i64 = dict(dtype=torch.int64, device=dev)
    ws_bytes = ctypes.c_size_t()
    _lib.call("hgt_plan_workspace_bytes", N, E, ctypes.byref(ws_bytes))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    dist = torch.empty(max(N, 1), **i32)
    hop_perm = torch.empty(max(n_rows, 1), **i32)
    hop_rank = torch.empty(max(N, 1), **i32)
    hop_nt = torch.empty(n_rows, **i64)
    hop_ei = torch.empty((2, E), **i64)
    out_rows = torch.empty(n_out, **i64)
    n_counts = T * (L + 2)
    head = (nt.data_ptr(), N, E, T, R, on.data_ptr(), n_out, L)
    tail = (dist.data_ptr(), hop_perm.data_ptr(), hop_rank.data_ptr(), hop_nt.data_ptr(), hop_ei.data_ptr(),
            out_rows.data_ptr())
    if bounds is None:
        meta = torch.empty(n_counts + T * R + 4, **i32)
        _lib.call("hgt_trim_layout", ei.data_ptr(), et.data_ptr(), _lib.ptr(tm), *head, *tail, meta.data_ptr(),
                  ws.data_ptr(), ws.numel(), st)
    else:
        meta = torch.empty(2 * n_counts + T * R + 6, **i32)
        b = np.ascontiguousarray(bounds, dtype=np.int32)
        _lib.call("hgt_trim_layout_bounded", ei.data_ptr(), et.data_ptr(), _lib.ptr(tm), *head, b.ctypes.data, n_rows,
                  *tail, meta.data_ptr(), ws.data_ptr(), ws.numel(), st)
    return dist[:N], hop_perm[:n_rows], hop_nt, hop_ei, out_rows, meta


def _raise_flags(flags, N):
    if flags[0]:
        raise IndexError("edge_index contains node ids outside [0, %d)" % N)
    if flags[1]:
        raise IndexError("edge_time contains values outside [0, %d) (RelTemporalEncoding table size)"
                         % _plan.RTE_MAX_LEN)
    if flags[2]:
        raise IndexError("out_nodes contains node ids outside [0, %d)" % N)


def build_layout(node_type, edge_index, edge_type, edge_time, out_nodes, num_types, num_relations, n_layers,
                 signature=None, pairs=None):
    nt, ei, et, tm, on = _check_args(node_type, edge_index, edge_type, edge_time, out_nodes)
    T, R, L = int(num_types), int(num_relations), int(n_layers)
    N = nt.numel()
    n_counts = T * (L + 2)
    if signature is None:
        # the read-back build: the exact counts become the slot sizes, so the layout has one row per node
        dist, hop_perm, hop_nt, hop_ei, out_rows, meta = _launch(nt, ei, et, tm, on, T, R, L)
        meta_h = meta.cpu().numpy()                          # the one host read-back of a trimmed forward
        _raise_flags(meta_h[n_counts + T * R:], N)
        counts = meta_h[:n_counts].reshape(T, L + 2).astype(np.int64)
        presence = meta_h[n_counts:n_counts + T * R].reshape(T, R)
        pairs = [(s, r) for s in range(T) for r in range(R) if presence[s, r]]
        bounds, n_other, flags = counts, N - int(counts.sum()), None
    else:
        if signature.num_types != T or signature.n_layers != L:
            raise ValueError("TrimSignature is for %d types and %d layers, the model has %d and %d"
                             % (signature.num_types, signature.n_layers, T, L))
        if pairs is None:
            raise ValueError("a TrimSignature layout needs the batch's <source type, relation> pairs")
        if N == 0:
            raise IndexError("out_nodes contains node ids outside [0, 0)")
        counts, bounds, n_other = None, signature.hop_bounds, 1
        dist, hop_perm, hop_nt, hop_ei, out_rows, meta = _launch(nt, ei, et, tm, on, T, R, L, bounds)
        flags = meta[n_counts + T * R:n_counts + T * R + 4]
    type_rows, actives, kvs, adapter_rows = slot_prefixes(bounds)
    hop = _plan.build_plan(hop_nt, hop_ei, et, tm, T, R, {"type_count": type_rows + [n_other], "sorted": True,
                                                         "pairs": list(pairs)})
    layers = []
    for active, kv in zip(actives, kvs):
        kv_runs = tuple(((s, r), ((0, kv[s]),)) for (s, r) in hop.pairs)
        ranges = [(hop.type_row0[t], hop.type_row0[t] + active[t]) for t in range(T) if active[t] > 0]
        layers.append(LayerView(plan=_range_view(hop, ranges), active=active, kv_runs=kv_runs))
    return TrimLayout(n_layers=L, counts=counts, dist=dist, perm=hop_perm.long(), out_rows=out_rows, plan=hop,
                      layers=layers, adapter_rows=adapter_rows, bounds=bounds,
                      counts_dev=meta[:n_counts].view(T, L + 2), flags_dev=flags,
                      bad=None if flags is None else flags.any(),
                      gather=None if flags is None else hop_perm.clamp(max=N - 1).long(),
                      pad_rows=None if flags is None else (hop_perm == N).unsqueeze(1))


def slot_prefixes(bounds):
    """Host arithmetic of a layout from its per-(type, hop) slot rows [T, L+2]: the rows of every type, then per layer
    l = 1..L the leading rows of each type it computes (hop classes 0..L-l) and whose K'/V' rows it reads (0..L-l+1),
    and the rows the input adapter computes (0..L)."""
    bounds = np.asarray(bounds, dtype=np.int64)
    T, L = bounds.shape[0], bounds.shape[1] - 2
    cum = np.cumsum(bounds, 1)                               # cum[t, b]: rows of type t with dist <= b
    actives = [tuple(int(cum[t, L - l]) for t in range(T)) for l in range(1, L + 1)]
    kvs = [tuple(int(cum[t, L - l + 1]) for t in range(T)) for l in range(1, L + 1)]
    return [int(c) for c in cum[:, -1]], actives, kvs, tuple(int(cum[t, L]) for t in range(T))


def _range_view(plan, ranges):
    """`plan` with edge tiles over the destination row ranges only (hgt_plan_range_tiles, sync-free) and its own
    layer-table and source-index caches."""
    dev = plan.row_ptr.device
    i32 = dict(dtype=torch.int32, device=dev)
    N, E = plan.n_nodes, plan.n_edges
    n_rows = sum(b - a for a, b in ranges)
    rng = _plan._to_dev_async(np.asarray(ranges if ranges else [(0, 0)], dtype=np.int32).reshape(-1), dev)
    max_tiles, max_split, max_hubs = _plan.tile_bounds(N, E, len(ranges))
    tiles = torch.empty((max_tiles, 4), **i32)
    hubs = torch.empty((max_hubs, 4), **i32)
    counts = torch.zeros(4, **i32)
    ws_bytes = ctypes.c_size_t()
    _lib.call("hgt_plan_workspace_bytes", N, E, ctypes.byref(ws_bytes))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    _lib.call("hgt_plan_range_tiles", plan.row_ptr.data_ptr(), N, E, rng.data_ptr(), len(ranges), n_rows,
              _plan.TILE_TARGET_EDGES, _plan.TILE_SPLIT_EDGES, tiles.data_ptr(), max_tiles, hubs.data_ptr(),
              max_hubs, counts.data_ptr(), ws.data_ptr(), ws.numel(), _plan._stream())
    return dataclasses.replace(plan, tiles=tiles, n_tiles=max_tiles if n_rows > 0 else 0, n_split=max_split, hubs=hubs,
                               n_hubs=max_hubs if max_split > 0 else 0, tile_counts_dev=counts, dst_ranges=rng,
                               n_dst_ranges=len(ranges), _layer_tables={}, _source_index={})
