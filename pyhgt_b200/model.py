"""Model wrapper mirroring pyHGT/model.py:54-80 (``GNN``): per-type input adapter ``tanh(Linear_t(x))`` followed by a
stack of ``GeneralConv('hgt')`` layers — SURVEY.md §8(f) rank 1.  Parameter names match the reference
(``adapt_ws.{t}.{weight,bias}``, ``gcs.{l}.base_conv.*``) so reference checkpoints load.

The adapter is the same "per-type linear dispatch" as inside HGTConv and runs through the same C-ABI grouped GEMM
(``hgt_typed_linear``: tensor cores when in_dim >= 64 and n_hid % 16 == 0, fp32 SIMT otherwise); every layer shares
the one cached graph plan.  Under autograd the adapter uses the same GEMM with its native backward
(``autograd._TypedLinear``).

``node_feature`` may be float32 or bfloat16 (e.g. the batches of ``sample_subgraph(s)_cuda(..., feature_dtype=
torch.bfloat16)``).  bf16 features are the adapter GEMM's bf16 operand as they are (hgt_typed_linear_bf16a, and
hgt_typed_linear_bwd_bf16a for dW in training): no fp32 copy, no split.  A bf16 value is exactly the hi half of the
split-bf16 scheme with a zero lo half, so every output, loss and gradient equals that of ``node_feature.float()``
bitwise.  bf16 features take no gradient.
"""
import torch
import torch.nn as nn

from . import _lib
from . import plan as _plan
from .autograd import _DROPOUT_MODULES, _TanhDropout, bf16_matmuls, drop_seed, fused_drop_p, gemm_impl
from .conv import GeneralConv, HGTConv


class GNN(nn.Module):
    fused_dropout = False      # training: the adapter's tanh and dropout as one pass (hgt_tanh_dropout) that keeps a single
                               # [N, n_hid] tensor for the backward; the layers have their own HGTConv.fused_dropout

    def __init__(self, in_dim, n_hid, num_types, num_relations, n_heads, n_layers, dropout=0.2, conv_name='hgt',
                 prev_norm=False, last_norm=False, use_RTE=True):
        super().__init__()
        self.gcs = nn.ModuleList()
        self.num_types = num_types
        self.in_dim = in_dim
        self.n_hid = n_hid
        self.adapt_ws = nn.ModuleList()
        self.drop = nn.Dropout(dropout)
        for _ in range(num_types):
            self.adapt_ws.append(nn.Linear(in_dim, n_hid))
        for _ in range(n_layers - 1):
            self.gcs.append(GeneralConv(conv_name, n_hid, n_hid, num_types, num_relations, n_heads, dropout,
                                        use_norm=prev_norm, use_RTE=use_RTE))
        self.gcs.append(GeneralConv(conv_name, n_hid, n_hid, num_types, num_relations, n_heads, dropout,
                                    use_norm=last_norm, use_RTE=use_RTE))
        self._ptrs = {}
        for gc in self.gcs[:-1]:                                   # every layer but the last feeds another projection
            if isinstance(gc.base_conv, HGTConv) and type(gc.base_conv) is HGTConv:
                gc.base_conv.emit_split = True

    def _adapter_table(self, plan, dev, rows=None):
        """Grouped-GEMM table of the input adapter over the first rows[t] nodes of every type (default: all of them)."""
        rows = tuple(plan.type_count[:self.num_types] if rows is None else rows)
        key = ("adapter", self.in_dim, self.n_hid, rows)
        table = plan._layer_tables.get(key)
        if table is None:
            groups, cblocks = [], []
            for t in range(self.num_types):
                if rows[t]:
                    groups.append((plan.type_row0[t], rows[t], t * self.n_hid, 1, len(cblocks), 1))
                    cblocks.append((plan.type_row0[t] * self.n_hid, self.n_hid))
            table = plan._layer_tables[key] = _plan._pack_groups(groups, cblocks, dev)
        return table

    def _adapter_cuda(self, node_feature, plan, rows=None):
        conv0 = self.gcs[0].base_conv
        T = self.num_types
        dev, N = node_feature.device, plan.n_nodes
        st = torch.cuda.current_stream().cuda_stream
        x = node_feature.contiguous()
        if not plan.sorted_types and x.dtype == torch.bfloat16:
            x = x.index_select(0, plan.perm.long())
        elif not plan.sorted_types:
            xs = torch.empty_like(x)
            _lib.call("hgt_gather_rows", x.data_ptr(), plan.perm.data_ptr(), N, self.in_dim, xs.data_ptr(), st)
            x = xs
        table = self._adapter_table(plan, dev, rows)
        w_cat = torch.empty((T * self.n_hid, self.in_dim), dtype=torch.float32, device=dev)
        b_cat = torch.empty(T * self.n_hid, dtype=torch.float32, device=dev)
        wp = conv0._ptrs("adapt_w", [l.weight for l in self.adapt_ws], dev)
        bp = conv0._ptrs("adapt_b", [l.bias for l in self.adapt_ws], dev)
        _lib.call("hgt_concat_linears", wp.data_ptr(), bp.data_ptr(), T, self.n_hid, self.in_dim, w_cat.data_ptr(),
                  b_cat.data_ptr(), st)
        # unknown-type rows stay 0 (model.py:70), and so do the rows past `rows`
        res = torch.zeros((N, self.n_hid), dtype=torch.float32, device=dev)
        impl = gemm_impl(conv0.linear_impl, bf16_matmuls())
        conv0._typed_linear(x, self.in_dim, w_cat, b_cat, self.in_dim, self.n_hid, table, res, impl, st)
        n_known = plan.type_row0[T]
        p_fused = fused_drop_p(self)
        if p_fused:                                                              # model.py:75-76 in one pass, in place
            _lib.call("hgt_tanh_dropout", res.data_ptr(), n_known, N, self.n_hid, drop_seed(dev).data_ptr(), p_fused,
                      res.data_ptr(), st)
        else:
            res[:n_known].tanh_()                                                # model.py:75
        if not plan.sorted_types:
            res = res.index_select(0, plan.rank.long())
        return res

    def _adapter_autograd(self, node_feature, plan, rows=None):
        """Training path of the adapter: the same grouped GEMM with its native backward (autograd._TypedLinear)."""
        from .autograd import typed_linear
        conv0 = self.gcs[0].base_conv
        T, h = self.num_types, self.n_hid
        N = plan.n_nodes
        x = node_feature if plan.sorted_types else node_feature.index_select(0, plan.perm.long())
        table = self._adapter_table(plan, node_feature.device, rows)
        w_cat = torch.cat([l.weight for l in self.adapt_ws], 0)
        b_cat = torch.cat([l.bias for l in self.adapt_ws], 0)
        n_known = plan.type_row0[T]
        zero = [((plan.type_row0[t] + rows[t]) * h, plan.type_row0[t + 1] * h) for t in range(T)] if rows else []
        res = typed_linear(x, w_cat, b_cat, table, h, N * h, gemm_impl(conv0.linear_impl, bf16_matmuls()), 0,
                           zero + [(n_known * h, N * h)]).view(N, h)
        _DROPOUT_MODULES.add(self)
        p_fused = fused_drop_p(self)
        if p_fused:                                                              # model.py:75-76 in one pass
            res = _TanhDropout.apply(res, n_known, drop_seed(res.device), p_fused)
        else:
            res = torch.cat([torch.tanh(res[:n_known]), res[n_known:]], 0) if n_known < N else torch.tanh(res)   # model.py:75
        if not plan.sorted_types:
            res = res.index_select(0, plan.rank.long())
        return res

    def forward(self, node_feature, node_type, edge_time, edge_index, edge_type, *, out_nodes=None, trim_signature=None):
        """pyHGT/model.py:64-80.  `out_nodes` (optional): 1-D int64 CUDA tensor of node ids (original order, duplicates
        allowed).  The call then returns only those rows, ``[len(out_nodes), n_hid]``, equal to ``forward(...)[out_nodes]``,
        and computes every layer only over the nodes the requested rows depend on (trim.py: layer l of L over the nodes
        within L - l hops of an out_nodes entry).  Inference and training both take this path; each layer's ``.att`` is
        then None.  In train mode dropout still applies, but its masks are drawn over the trimmed shapes, so they differ
        from those of the untrimmed call.  Only 'hgt' layers support it ('dense_hgt' raises ValueError).

        `trim_signature` (optional, with out_nodes): a trim.TrimSignature.  The layout of a new batch is then built
        without reading anything back (its pairs come from the batch's cached plan, which sample_subgraph(s)_cuda,
        merge_batches and the graphed classes leave), so the call can be captured in a CUDA graph.  Rows are padded to
        the bounds; padding changes no real row.  If a (type, hop) class of the batch exceeds its bound or an out_nodes id
        is out of range, every returned row is NaN and the layout's check() raises (trim.get_layout(...).check()).

        `node_feature` is float32 or bfloat16 (ValueError otherwise); bf16 features must not require grad."""
        grad = torch.is_grad_enabled() and (node_feature.requires_grad or any(p.requires_grad for p in self.parameters()))
        if not node_feature.is_cuda:
            raise _lib.HgtError("pyhgt_b200.GNN runs on CUDA tensors only (got %s): there is no CPU fallback"
                                % node_feature.device)
        if node_feature.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("node_feature must be float32 or bfloat16, got %s" % (node_feature.dtype,))
        if node_feature.dtype == torch.bfloat16 and node_feature.requires_grad:
            raise ValueError("bf16 node_feature cannot require grad: features are data, and the adapter offers no bf16 "
                             "input gradient")
        if out_nodes is not None:
            return self._forward_trimmed(node_feature, node_type, edge_time, edge_index, edge_type, out_nodes, grad,
                                         trim_signature)
        if trim_signature is not None:
            raise ValueError("trim_signature needs out_nodes")
        conv0 = self.gcs[0].base_conv
        plan = _plan.get_plan(node_type, edge_index, edge_type, edge_time if conv0.use_RTE else None, self.num_types,
                              conv0.num_relations)
        res = self._adapter_autograd(node_feature, plan) if grad else self._adapter_cuda(node_feature, plan)
        meta_xs = res if fused_drop_p(self) else self.drop(res)                  # fused: the adapter already dropped
        del res
        for gc in self.gcs:
            meta_xs = gc(meta_xs, node_type, edge_index, edge_type, edge_time)
        return meta_xs

    def _forward_trimmed(self, node_feature, node_type, edge_time, edge_index, edge_type, out_nodes, grad, tsig=None):
        from . import trim
        if any(type(gc.base_conv) is not HGTConv for gc in self.gcs):
            raise ValueError("GNN.forward(out_nodes=) supports conv_name='hgt' only")
        if not out_nodes.is_cuda:
            raise _lib.HgtError("out_nodes must be a CUDA tensor (got %s): there is no CPU fallback" % out_nodes.device)
        if node_feature.dim() != 2 or node_feature.shape[0] != node_type.numel():
            raise ValueError("node_feature must be [N, in_dim] with N = len(node_type), got %s"
                             % (tuple(node_feature.shape),))
        if out_nodes.numel() == 0:
            return node_feature.new_zeros((0, self.n_hid), dtype=torch.float32)
        conv0 = self.gcs[0].base_conv
        tm = edge_time if conv0.use_RTE else None
        pairs = None
        if tsig is not None:
            # the pairs of the batch's cached plan (a batch without one costs one read-back here)
            pairs = _plan.get_plan(node_type, edge_index, edge_type, tm, self.num_types, conv0.num_relations).pairs
        lay = trim.get_layout(node_type, edge_index, edge_type, tm, out_nodes, self.num_types, conv0.num_relations,
                              len(self.gcs), tsig, pairs)
        if lay.padded:                                                           # hop order; padding rows are zero
            x = node_feature.index_select(0, lay.gather).masked_fill_(lay.pad_rows, 0.0)
        else:
            x = node_feature.index_select(0, lay.perm)                           # hop order
        if grad:
            res = self._adapter_autograd(x, lay.plan, lay.adapter_rows)
        else:
            res = self._adapter_cuda(x, lay.plan, lay.adapter_rows)
        meta_xs = res if fused_drop_p(self) else self.drop(res)
        del res
        for gc, view in zip(self.gcs, lay.layers):
            meta_xs = gc.base_conv._forward_view(meta_xs, view, edge_time)
        out = meta_xs.index_select(0, lay.out_rows)
        if lay.padded:                                          # overflow / bad ids: NaN rows instead of a host sync
            out = torch.where(lay.bad, torch.full_like(out, float("nan")), out)
        return out
