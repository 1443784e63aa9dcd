"""Training path of pyhgt_b200.HGTConv (reference: the same forward differentiated by autograd,
OAG/train_paper_field.py:249 ``loss.backward()``).

Every stage is a custom autograd.Function whose forward AND backward are hand-written kernels behind the C ABI:

    _FoldWeights     hgt_fold_weights / hgt_fold_backward        relation_att/msg/pri folded into the typed K/V weights
    _TypedLinear     hgt_act_split + hgt_typed_linear_presplit   typed projections, a_linears, RTE tables (wgmma
                     / hgt_typed_linear_bwd                      split-bf16 forward, dX and dW; fp32 SIMT for odd shapes);
                                                                 the gelu in front of the a_linears (conv.py:119) lives in
                                                                 the operand split (forward) and the dX epilogue (backward)
    _EdgeAttention   hgt_edge_forward / hgt_edge_backward        score -> softmax by destination -> weighted aggregation;
                                                                 att is differentiable: a loss term on it takes the
                                                                 hgt_edge_att_grad_prep + hgt_edge_backward*_att calls
    _UpdateEpilogue  hgt_update_epilogue / hgt_update_backward   sigmoid(skip) gate + LayerNorm (conv.py:129-133)

No per-edge intermediates are kept: the edge backward recomputes the softmax weights from the saved per-destination
(max, sum); the typed linears keep the bf16 hi/lo split of their input (the A operand of the dW product).  No cuBLAS,
no torch matmul on this path.  Gradients reach ``node_inp`` and every parameter of conv.py:28-54 including ``emb.*``.
The inference path (``torch.no_grad``) does not come through here: it uses the fused kernels in conv.py.

Under ``torch.use_deterministic_algorithms(True)`` (``warn_only=True`` included) every stage records the flag in its
forward and its backward calls the deterministic twins instead: hgt_edge_backward_dst + hgt_edge_backward_rows (a
source-major second pass that owns every K'/V' and RTE gradient row, plan.source_index), hgt_typed_linear_bwd_det,
hgt_update_backward_det and hgt_fold_backward_det.  They use no float atomics, so two identical steps give bitwise equal
gradients.  With the flag off nothing changes.

With ``HGTConv.fused_dropout`` (and ``GNN.fused_dropout`` for the input adapter) training dropout is drawn inside the
update kernels instead of by ``nn.Dropout``: _UpdateEpilogue takes (seed, p), hgt_update_epilogue_drop scales ``o`` by a
counter-based mask as it loads the row, and hgt_update_backward_drop[_det] regenerates the mask from the saved one-element
seed tensor.  The saved ``o`` is the pre-dropout tensor; no mask and no dropped copy exist.  The masks are a different
random stream from ``nn.Dropout``'s, which is why the switch is off by default (mask contract: include/hgt_b200.h).

Under ``torch.autocast("cuda", dtype=torch.bfloat16)`` (bf16_tables()) the two gathered tables, [K'|V'] and the RTE table
KVR, are stored in bf16: the projection writes Q by its own fp32 call and the K'/V' blocks straight into the bf16 table
(hgt_typed_linear[_presplit]_bf16, rounded once from the fp32 accumulator), and the edge kernels read them through their
_bf16 entry points.  The layer output, att, the softmax statistics, Q and every gradient stay fp32; the stages record the
switch on ctx, so the backward follows the forward.  fp16 autocast keeps fp32 tables.

Under ``torch.set_float32_matmul_precision("medium")`` (bf16_matmuls()) the typed GEMMs that would run on the tensor cores
(linear_impl 0 or 2) run with one bf16 product instead of the split-bf16 x3 (C impl 3): the operands are rounded to bf16
and only that hi half is produced, saved for dW and read.  This is torch's documented meaning of "medium" ("bfloat16
datatype for internal computations"); note that torch's own CUDA matmuls run TF32 at "medium", so these GEMMs are less
precise than torch's there.  "high" and "highest" keep the x3 scheme.  The stages record the setting on ctx.
"""
import ctypes
import weakref

import numpy as np
import torch

from . import _lib
from . import plan as _plan


def _stream():
    return torch.cuda.current_stream().cuda_stream


def fused_drop_p(m):
    """Drop probability of module `m` (a layer or the GNN) when its dropout is drawn inside the kernels, else 0."""
    return float(m.drop.p) if (m.training and m.drop.p > 0 and m.fused_dropout) else 0.0


def drop_seed(dev):
    """One 64-bit Philox key for one dropout site of one forward, drawn on the device from torch's CUDA generator: it
    follows torch.manual_seed, needs no host read-back, and inside a CUDA graph every replay draws a new one."""
    return torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=dev)


# layers whose .att is still a node of the last training step's autograd graph (it keeps that graph alive)
_ATT_GRAPH_LAYERS = weakref.WeakSet()


def _set_att(m, att):
    m.att = att
    if att is not None and att.requires_grad:
        _ATT_GRAPH_LAYERS.add(m)


def release_att_graphs(params):
    """Detach `.att` of the layers that own one of `params` and whose att still holds an autograd graph.  That graph
    keeps the parameters' AccumulateGrad nodes alive, and the next step would reuse them on the stream they were made
    on; graphed.py calls this for the parameters of the step it captures, before and after the capture.  Layers of
    other models keep their att (and a loss term on it that has not run backward yet)."""
    owned = {id(p) for p in params}
    for m in list(_ATT_GRAPH_LAYERS):
        if any(id(p) in owned for p in m.parameters()):
            if m.att is not None:
                m.att = m.att.detach()
            _ATT_GRAPH_LAYERS.discard(m)


def bf16_tables():
    """The switch for bf16 gather tables, read once per layer forward: bf16 autocast on CUDA."""
    return torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


def bf16_matmuls():
    """The switch for one bf16 product in the tensor-core GEMMs, read once per layer forward:
    torch.get_float32_matmul_precision() == "medium"."""
    return torch.get_float32_matmul_precision() == "medium"


def gemm_impl(linear_impl, one_product):
    """The C `impl` of a layer's typed GEMMs: 3 (auto, one bf16 product on the tensor cores) where the layer would take
    the tensor cores (linear_impl 0 or 2) and one_product is set; linear_impl otherwise (1 keeps fp32 SIMT)."""
    return 3 if one_product and linear_impl in (0, 2) else linear_impl


def _tc_shape_ok(K, width):
    """Shapes both the tensor-core forward (hgt_typed_linear_presplit) and backward (hgt_typed_linear_bwd) take."""
    return K % 16 == 0 and K >= 64 and width % 16 == 0


class _TypedLinear(torch.autograd.Function):
    """out_flat[cblock c of group g][m, :] = act(A)[rows_g] @ W_cat[rows of (g, c)]^T + b_cat   (act: 0 none, 1 gelu).

    tables16 (bf16 gather tables) = (q_table or None, q_elems, kv_table, kv_off, kv_zero_ranges): the same product split
    into an fp32 Q buffer [q_elems] (q_table) and a bf16 table [out_elems - kv_off] (kv_table, offsets relative to kv_off,
    zero ranges relative to it too).  The forward then returns (stand-in, q, table): the stand-in is a zero-stride fp32
    tensor of out_elems that only carries the gradient, which arrives in the flat layout of the fp32 output, so the
    backward is the same.  impl 3: one bf16 product on the tensor cores, only the hi half of act(A) is made and saved.

    A bf16 `a` (the input adapter fed bf16 features; act 0, fp32 output, no gradient for a): the GEMM reads it as its
    bf16 operand (hgt_typed_linear_bf16a) and it is saved as it is for dW (hgt_typed_linear_bwd_bf16a): no split, no lo
    half, no fp32 copy.  Output, dW and db are bitwise those of the fp32 `a.float()`."""

    @staticmethod
    def forward(ctx, a, w_cat, b_cat, table, width, out_elems, impl, act, zero_ranges, tables16=None):
        a = a.contiguous()
        w_cat = w_cat.contiguous()
        K = a.shape[1]
        use_tc = impl in (0, 2, 3) and _tc_shape_ok(K, width)
        one = use_tc and impl == 3
        ctx.bf16a = a.dtype == torch.bfloat16
        if ctx.bf16a:
            if act or tables16 is not None or a.requires_grad:
                raise ValueError("a bf16 typed-linear input takes no activation, no bf16 tables and no gradient")
            out = _linear_outputs(out_elems, zero_ranges, None, a.device)[0]
            _linear_gemm_bf16a(a, w_cat, b_cat, table, width, (3 if one else 2) if use_tc else 1, out)
            ctx.table, ctx.width, ctx.has_bias, ctx.act, ctx.use_tc = table, width, b_cat is not None, 0, use_tc
            ctx.one = one
            ctx.out_elems = out_elems
            ctx.det = torch.are_deterministic_algorithms_enabled()
            ctx.save_for_backward(a, w_cat)
            return out
        out, q, kv = _linear_outputs(out_elems, zero_ranges, tables16, a.device)
        hi, lo, a_act = _split_operand(a, act, use_tc, one)
        _linear_gemms(hi, lo, a_act, w_cat, b_cat, table, width, use_tc, tables16, out, q, kv)
        ctx.table, ctx.width, ctx.has_bias, ctx.act, ctx.use_tc = table, width, b_cat is not None, act, use_tc
        ctx.one = one
        ctx.out_elems = out_elems
        ctx.det = torch.are_deterministic_algorithms_enabled()
        # gelu'(a) needs the un-activated input; the dW product needs act(a): as the bf16 split (tensor cores) or fp32
        ctx.save_for_backward(a if (act or not use_tc) else None, a_act if (act and not use_tc) else None, hi, lo, w_cat)
        if tables16 is None:
            return out
        ctx.mark_non_differentiable(*[t for t in (q, kv) if t is not None])
        return torch.zeros(1, dtype=torch.float32, device=a.device).expand(out_elems), q, kv

    @staticmethod
    def backward(ctx, dout, *_unused):
        if ctx.bf16a:
            a, w_cat = ctx.saved_tensors
            dw, db = _linear_backward_bf16a(ctx, dout, a, w_cat)
            return None, dw, db, None, None, None, None, None, None, None
        a, a_act, hi, lo, w_cat = ctx.saved_tensors
        da, dw, db = _linear_backward(ctx, dout, a, a_act, hi, lo, w_cat, ctx.needs_input_grad[0])
        return da, dw, db, None, None, None, None, None, None, None


def _linear_gemm_bf16a(a, w_cat, b_cat, table, width, impl, out):
    """out = a @ w_cat^T + b_cat over the table's groups for a bf16 `a` (hgt_typed_linear_bf16a, C impl `impl`)."""
    K = a.shape[1]
    g_dev, g_host, n_g, c_dev = table
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=a.device)
    _lib.call("hgt_typed_linear_bf16a", a.data_ptr(), K, w_cat.data_ptr(), _lib.ptr(b_cat), K, width, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), out.data_ptr(), impl, ws.data_ptr(), ws.numel(), _stream())


def _linear_backward_bf16a(ctx, dout, a, w_cat):
    """dW, db of _TypedLinear with a bf16 `a`: hgt_typed_linear_bwd_bf16a[_det] with `a` as the dW operand."""
    width = ctx.width
    K = w_cat.shape[1]
    dout = dout.contiguous()
    dw = torch.zeros_like(w_cat)
    db = torch.zeros(w_cat.shape[0], dtype=torch.float32, device=w_cat.device) if ctx.has_bias else None
    impl = (3 if ctx.one else 2) if ctx.use_tc else 1
    sfx = "_det" if ctx.det else ""
    g_dev, g_host, n_g, _ = ctx.table
    c_host = ctx.table.c_host
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_bwd" + sfx + "_workspace_bytes", g_host.ctypes.data, n_g, c_host.ctypes.data, K, width,
              K, ctx.out_elems, 0, 1, impl, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=w_cat.device)
    _lib.call("hgt_typed_linear_bwd_bf16a" + sfx, dout.data_ptr(), ctx.out_elems, a.data_ptr(), K, K, width,
              g_dev.data_ptr(), g_host.ctypes.data, n_g, c_host.ctypes.data, dw.data_ptr(), _lib.ptr(db), impl,
              ws.data_ptr(), ws.numel(), _stream())
    return dw, db


def _split_operand(a, act, use_tc, one):
    """act(a) as the typed GEMM reads it: (hi, lo, a_act), the bf16 hi/lo split on the tensor cores (hi only for one
    bf16 product) or a_act, fp32 act(a), on the SIMT path."""
    rows, K = a.shape
    dev = a.device
    st = _stream()
    hi = lo = a_act = None
    if use_tc:
        hi = torch.empty((rows, K), dtype=torch.bfloat16, device=dev)
        lo = None if one else torch.empty((rows, K), dtype=torch.bfloat16, device=dev)
        _lib.call("hgt_act_split", a.data_ptr(), K, rows, K, act, None, hi.data_ptr(), _lib.ptr(lo), st)
    else:
        a_act = a
        if act:
            a_act = torch.empty_like(a)
            _lib.call("hgt_act_split", a.data_ptr(), K, rows, K, act, a_act.data_ptr(), None, None, st)
    return hi, lo, a_act


def _linear_outputs(out_elems, zero_ranges, tables16, dev):
    """The output buffers of _TypedLinear: (out, None, None), or (None, q or None, kv) with tables16."""
    out = q = kv = None
    if tables16 is None:
        out = torch.empty(out_elems, dtype=torch.float32, device=dev)
        for (z0, z1) in zero_ranges:                                   # padding / all-zero table rows only
            if z1 > z0:
                out[z0:z1].zero_()
    else:
        q_table, q_elems, kv_table, kv_off, kv_zero = tables16
        q = torch.empty(q_elems, dtype=torch.float32, device=dev) if q_table is not None else None
        kv = torch.empty(out_elems - kv_off, dtype=torch.bfloat16, device=dev)
        for (z0, z1) in kv_zero:
            if z1 > z0:
                kv[z0:z1].zero_()
    return out, q, kv


def _linear_gemms(hi, lo, a_act, w_cat, b_cat, table, width, use_tc, tables16, out, q, kv):
    """The forward product of _TypedLinear on its split operand into the buffers of _linear_outputs.  The GEMMs are
    deterministic: the same call on the same operands writes the same outputs bit for bit."""
    K = w_cat.shape[1]
    dev = w_cat.device
    st = _stream()

    def gemm(tab, dst):
        g_dev, g_host, n_g, c_dev = tab
        sfx = "_bf16" if dst.dtype == torch.bfloat16 else ""
        wsb = ctypes.c_size_t()
        if use_tc:
            _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
            ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
            _lib.call("hgt_typed_linear_presplit" + sfx, hi.data_ptr(), _lib.ptr(lo), w_cat.data_ptr(),
                      _lib.ptr(b_cat), K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(),
                      dst.data_ptr(), ws.data_ptr(), ws.numel(), st)
        else:
            _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, 1, ctypes.byref(wsb))
            ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
            _lib.call("hgt_typed_linear" + sfx, a_act.data_ptr(), K, w_cat.data_ptr(), _lib.ptr(b_cat), K, width,
                      g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), dst.data_ptr(), 1, ws.data_ptr(),
                      ws.numel(), st)

    if tables16 is None:
        gemm(table, out)
    else:
        if q is not None:
            gemm(tables16[0], q)
        gemm(tables16[2], kv)


def _linear_backward(ctx, dout, a, a_act, hi, lo, w_cat, need_da):
    """dA, dW, db of _TypedLinear from the gradient of its flat output; ctx carries the forward's table, width,
    has_bias, act, use_tc, one, out_elems and det."""
    width = ctx.width
    K = w_cat.shape[1]
    dev = w_cat.device
    rows = hi.shape[0] if hi is not None else a.shape[0]
    dout = dout.contiguous()
    da = torch.empty((rows, K), dtype=torch.float32, device=dev) if need_da else None
    dw = torch.zeros_like(w_cat)                                       # small: [sum of out rows, K]
    db = torch.zeros(w_cat.shape[0], dtype=torch.float32, device=dev) if ctx.has_bias else None
    impl = (3 if ctx.one else 2) if ctx.use_tc else 1
    fn = "hgt_typed_linear_bwd_det" if ctx.det else "hgt_typed_linear_bwd"
    a_f32 = a_act if a_act is not None else a                          # SIMT dW operand (act already applied)
    # tables whose groups overlap in rows (sharded per-pair compaction) come with disjoint sub-tables: the first call
    # writes dA, the others accumulate into it; dW / db accumulate anyway
    tables = getattr(ctx.table, "bwd_tables", None) or [ctx.table]
    if not ctx.use_tc:
        tables = [ctx.table]                                           # the SIMT dX adds overlapping groups itself
    if need_da:
        # hgt_typed_linear_bwd zeroes the gaps between the first table's groups; rows past its last group (other
        # sub-tables' rows, nodes of unknown type) are zeroed here
        g0, n0 = tables[0][1], tables[0][2]
        end0 = int((g0["a_row0"][:n0] + g0["m"][:n0]).max()) if n0 else 0
        if end0 < rows:
            da[end0:].zero_()
    for ti, tab in enumerate(tables):
        g_dev, g_host, n_g, _ = tab
        c_host = tab.c_host
        wsb = ctypes.c_size_t()
        _lib.call(fn + "_workspace_bytes", g_host.ctypes.data, n_g, c_host.ctypes.data, K, width, K,
                  ctx.out_elems, 0, int(hi is not None), impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        _lib.call(fn, dout.data_ptr(), None, None, ctx.out_elems, _lib.ptr(a_f32), K, _lib.ptr(hi),
                  _lib.ptr(lo), w_cat.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g,
                  c_host.ctypes.data, _lib.ptr(da), int(ti > 0), a.data_ptr() if ctx.act else None, dw.data_ptr(),
                  _lib.ptr(db), impl, ws.data_ptr(), ws.numel(), _stream())
    return da, dw, db


class _EdgeAttention(torch.autograd.Function):
    """agg[i] = sum_{e -> i} softmax_i(<Q[i], K'[e]>) * V'[e]   (conv.py:99,108-111 + scatter-add).  Takes and returns
    the FLAT projection buffer (Q at q_off, the [K'|V'] table at kv_off): its gradient is produced as one buffer, so
    autograd never assembles it from slices.  tables16 (bf16 gather tables): (Q, bf16 [K'|V'] table, bf16 RTE table or
    None) from _TypedLinear; proj / kvr are then its stand-ins and receive the fp32 gradients in the same layouts."""

    @staticmethod
    def forward(ctx, proj, kvr, plan, lt, d, n_heads, want_att, variant, tables16=None):
        N = plan.n_nodes
        ctx.bf16 = tables16 is not None
        if ctx.bf16:
            q, kv, kvr = tables16
        else:
            proj = proj.contiguous()
            q = proj[lt.q_off:lt.q_off + N * d]
            kv = proj[lt.kv_off:]
            kvr = None if kvr is None else kvr.contiguous()
        agg, att, stats = _edge_forward(q, kv, kvr, plan, lt, d, n_heads, want_att, variant, ctx.bf16)
        ctx.plan, ctx.lt, ctx.d, ctx.n_heads, ctx.has_kvr = plan, lt, d, n_heads, kvr is not None
        ctx.det = torch.are_deterministic_algorithms_enabled()
        ctx.proj_elems = proj.numel()
        # att is differentiable (conv.py:108 makes it a node of the graph): a loss term on it arrives as datt.  Without
        # materialised grads an unused att gives datt None, and the backward runs exactly the calls without it.
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(q, kv, kvr, agg, stats, att)
        return agg, att

    @staticmethod
    def backward(ctx, dagg, datt=None):
        q, kv, kvr, agg, stats, att = ctx.saved_tensors
        plan, lt, d, H = ctx.plan, ctx.lt, ctx.d, ctx.n_heads
        N = plan.n_nodes
        f32 = dict(dtype=torch.float32, device=q.device)
        if dagg is None:                                               # the loss reads att only
            dagg = torch.zeros((N, d), **f32)
        dproj = torch.empty(ctx.proj_elems, **f32)                     # hgt_edge_backward zero-initialises dq / dkv
        if lt.kv_off > N * d:
            dproj[N * d:lt.kv_off].zero_()                             # alignment gap
        dq = dproj[lt.q_off:lt.q_off + N * d]
        dkv = dproj[lt.kv_off:]
        dkvr = torch.empty(kvr.numel(), **f32) if kvr is not None else None
        dagg = dagg.contiguous()
        sfx = "_bf16" if ctx.bf16 else ""
        att_grad = _att_grad_prep(att, datt, plan, H) if datt is not None else None
        if ctx.det:
            _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, sfx, att_grad)
            return dproj, dkvr, None, None, None, None, None, None, None
        ws = torch.empty(256, dtype=torch.uint8, device=q.device)
        fn, extra = "hgt_edge_backward", ()
        if att_grad is not None:
            fn, extra = "hgt_edge_backward_att", (att_grad[0].data_ptr(), att_grad[1].data_ptr())
        _lib.call(fn + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(), dagg.data_ptr(),
                  stats.data_ptr(), *extra, plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
                  None if kvr is None else plan.rte_row.data_ptr(), plan.tiles.data_ptr(), plan.n_tiles, N, d, H,
                  plan.kv_rows + 1, 0 if kvr is None else kvr.numel() // (2 * d),
                  dq.data_ptr(), dkv.data_ptr(), _lib.ptr(dkvr), ws.data_ptr(), ws.numel(),
                  _lib.ptr(plan.tile_counts_dev), _stream())
        return dproj, dkvr, None, None, None, None, None, None, None


def _edge_forward(q, kv, kvr, plan, lt, d, n_heads, want_att, variant, bf16):
    """hgt_edge_forward[_bf16]: (agg [N, d], att [E, H] or None, softmax statistics [N, 2H])."""
    N = plan.n_nodes
    dev = q.device
    ws_bytes = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, n_heads, ctypes.byref(ws_bytes))
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
    agg = torch.empty((N, d), dtype=torch.float32, device=dev)
    stats = torch.empty((N, 2 * n_heads), dtype=torch.float32, device=dev)
    att = torch.empty((plan.n_edges, n_heads), dtype=torch.float32, device=dev) if want_att else None
    _lib.call("hgt_edge_forward_bf16" if bf16 else "hgt_edge_forward", q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), plan.row_ptr.data_ptr(),
              plan.kv_row.data_ptr(), None if kvr is None else plan.rte_row.data_ptr(), plan.csr_eid.data_ptr(),
              plan.tiles.data_ptr(), plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, N, plan.n_edges, d,
              n_heads, 0, agg.data_ptr(), _lib.ptr(att), stats.data_ptr(), None, None, ws.data_ptr(), ws.numel(),
              variant, _lib.ptr(plan.tile_counts_dev), plan.type_row0_dev.data_ptr(), plan.num_types,
              _lib.ptr(lt.type_active_dev), _stream())
    return agg, att, stats


def _att_grad_prep(att, datt, plan, H):
    """(datt in CSR order [E, H], C [N, H]) for the *_att backward calls: hgt_edge_att_grad_prep."""
    dev = att.device
    datt = datt.contiguous()
    datt_csr = torch.empty((max(plan.n_edges, 1), H), dtype=torch.float32, device=dev)
    c_att = torch.empty((plan.n_nodes, H), dtype=torch.float32, device=dev)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_att_grad_workspace_bytes", plan.n_split, H, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    _lib.call("hgt_edge_att_grad_prep", att.data_ptr(), datt.data_ptr(), plan.csr_eid.data_ptr(), plan.row_ptr.data_ptr(),
              plan.tiles.data_ptr(), plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, plan.n_nodes, H,
              c_att.data_ptr(), datt_csr.data_ptr(), ws.data_ptr(), ws.numel(), _lib.ptr(plan.tile_counts_dev), _stream())
    return datt_csr, c_att


def _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, sfx="", att_grad=None, rte_first=False):
    """Deterministic edge backward: destination pass (dq, D), then one row pass over the [K'|V'] rows and, with RTE, one
    over the RTE rows; each gradient row is written once by its owner.  sfx "_bf16": bf16 kv / kvr tables.  att_grad:
    None, or (datt_csr, C) from _att_grad_prep: the *_att passes, the row passes reading datt at the CSR positions the
    source-major indices carry (plan.source_index(..., with_pos=True)).  rte_first: the RTE row pass, which reads the
    K'/V' rows, runs before the K'/V' pass, so that dkv may be kv itself (fp32 tables; _ProjectEdgeLean)."""
    N = plan.n_nodes
    st = _stream()
    with_pos = att_grad is not None
    kvi = _plan.source_index(plan, "kv", with_pos)
    rti = _plan.source_index(plan, "rte", with_pos) if kvr is not None else None
    D = torch.empty((N, H), dtype=torch.float32, device=q.device)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_backward_det_workspace_bytes", plan.n_split, max(kvi.n_split, rti.n_split if rti else 0), d,
              ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=q.device)
    att_sfx, dst_extra = "", ()
    if att_grad is not None:
        att_sfx, dst_extra = "_att", (att_grad[0].data_ptr(), att_grad[1].data_ptr())
    _lib.call("hgt_edge_backward_dst" + att_sfx + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(),
              dagg.data_ptr(), stats.data_ptr(), *dst_extra, plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
              None if kvr is None else plan.rte_row.data_ptr(), plan.tiles.data_ptr(), plan.n_tiles, plan.n_split,
              plan.hubs.data_ptr(), plan.n_hubs, N, d, H, dq.data_ptr(), D.data_ptr(), ws.data_ptr(), ws.numel(),
              _lib.ptr(plan.tile_counts_dev), st)
    passes = [(kv, kvr, kvi, plan.kv_rows + 1, dkv)]
    if kvr is not None:
        passes.append((kvr, kv, rti, kvr.numel() // (2 * d), dkvr))
    if rte_first:
        passes.reverse()
    for own, oth, idx, own_rows, grad in passes:
        src_oth = None if oth is None else idx.oth.data_ptr()
        if att_grad is None:
            _lib.call("hgt_edge_backward_rows" + sfx, q.data_ptr(), dagg.data_ptr(), stats.data_ptr(), D.data_ptr(),
                      own.data_ptr(), _lib.ptr(oth), idx.ptr.data_ptr(), idx.dst.data_ptr(), src_oth,
                      idx.n_rows, own_rows, idx.tiles.data_ptr(), idx.n_tiles, idx.n_split, idx.hubs.data_ptr(),
                      idx.n_hubs, d, H, grad.data_ptr(), ws.data_ptr(), ws.numel(), idx.counts_dev.data_ptr(), st)
        else:
            _lib.call("hgt_edge_backward_rows_att" + sfx, q.data_ptr(), dagg.data_ptr(), stats.data_ptr(), D.data_ptr(),
                      att_grad[0].data_ptr(), own.data_ptr(), _lib.ptr(oth), idx.ptr.data_ptr(), idx.dst.data_ptr(),
                      src_oth, idx.pos.data_ptr(), idx.n_rows, own_rows, idx.tiles.data_ptr(), idx.n_tiles, idx.n_split,
                      idx.hubs.data_ptr(), idx.n_hubs, d, H, grad.data_ptr(), ws.data_ptr(), ws.numel(),
                      idx.counts_dev.data_ptr(), st)


class _ProjectEdgeLean(torch.autograd.Function):
    """The typed projection and the edge attention of a layer as one stage that keeps neither Q nor the [K'|V'] table
    for the backward (HGTConv.recompute_tables).  The forward saves what the projection's own backward needs anyway (the
    bf16 split of x, or fp32 x on the SIMT path, and W_cat), b_cat, the RTE table and the edge kernel's outputs.  The
    backward
      1. recomputes the projection with the forward's GEMM calls on those operands: the same tables bit for bit;
      2. runs the destination pass: dq into its own [N, d] buffer, and D;
      3. with RTE, runs the RTE row pass into dkvr (it reads the K'/V' rows, so it goes before 4);
      4. runs the K'/V' row pass.  fp32 tables: each row's gradient is written over the row itself (hgt_edge_backward_rows
         accepts grad == own), then dq is copied over Q, which turns the recomputed buffer into its own gradient.  bf16
         tables: the fp32 gradient goes to its own buffer, as in _EdgeAttention;
      5. runs the projection backward (dX, dW, db) as _TypedLinear does.
    The edge passes are the source-major ones whatever the deterministic flag (only they can write in place); with the
    flag on the gradients are those of _TypedLinear + _EdgeAttention bit for bit.  kvr: the RTE table (fp32) or its
    gradient stand-in (bf16, kvr16 is then the table the kernels read)."""

    @staticmethod
    def forward(ctx, x, w_cat, b_cat, kvr, plan, lt, d, n_heads, want_att, variant, impl, bf16, kvr16):
        x = x.contiguous()
        w_cat = w_cat.contiguous()
        N, K = plan.n_nodes, x.shape[1]
        use_tc = impl in (0, 2, 3) and _tc_shape_ok(K, d)
        one = use_tc and impl == 3
        zero_ranges, tables16 = _proj_layout(plan, lt, d, bf16)
        out, q, kv = _linear_outputs(lt.proj_elems, zero_ranges, tables16, x.device)
        hi, lo, a_act = _split_operand(x, 0, use_tc, one)
        _linear_gemms(hi, lo, a_act, w_cat, b_cat, lt.proj_groups, d, use_tc, tables16, out, q, kv)
        if bf16:
            table = kvr16
        else:
            q, kv = out[lt.q_off:lt.q_off + N * d], out[lt.kv_off:]
            table = None if kvr is None else kvr.contiguous()
        agg, att, stats = _edge_forward(q, kv, table, plan, lt, d, n_heads, want_att, variant, bf16)
        # the attributes _linear_backward reads, as _TypedLinear records them
        ctx.table, ctx.width, ctx.has_bias, ctx.act, ctx.use_tc = lt.proj_groups, d, b_cat is not None, 0, use_tc
        ctx.one = one
        ctx.out_elems = lt.proj_elems
        ctx.det = torch.are_deterministic_algorithms_enabled()
        ctx.plan, ctx.lt, ctx.d, ctx.n_heads, ctx.bf16 = plan, lt, d, n_heads, bf16
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(None if use_tc else x, hi, lo, w_cat, b_cat, table, agg, stats, att)
        return agg, att

    @staticmethod
    def backward(ctx, dagg, datt=None):
        x, hi, lo, w_cat, b_cat, kvr, agg, stats, att = ctx.saved_tensors
        plan, lt, d, H = ctx.plan, ctx.lt, ctx.d, ctx.n_heads
        N = plan.n_nodes
        f32 = dict(dtype=torch.float32, device=agg.device)
        zero_ranges, tables16 = _proj_layout(plan, lt, d, ctx.bf16)
        out, q, kv = _linear_outputs(lt.proj_elems, zero_ranges, tables16, agg.device)
        _linear_gemms(hi, lo, x, w_cat, b_cat, lt.proj_groups, d, ctx.use_tc, tables16, out, q, kv)
        if dagg is None:                                               # the loss reads att only
            dagg = torch.zeros((N, d), **f32)
        dagg = dagg.contiguous()
        att_grad = _att_grad_prep(att, datt, plan, H) if datt is not None else None
        if ctx.bf16:
            dproj = torch.empty(lt.proj_elems, **f32)
            if lt.kv_off > N * d:
                dproj[N * d:lt.kv_off].zero_()                         # alignment gap
            dq, dkv = dproj[lt.q_off:lt.q_off + N * d], dproj[lt.kv_off:]
        else:
            q, kv = out[lt.q_off:lt.q_off + N * d], out[lt.kv_off:]
            dproj, dq, dkv = out, torch.empty(N * d, **f32), kv        # the gap and the zero row stay zero
        dkvr = torch.empty(kvr.numel(), **f32) if kvr is not None else None
        _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, "_bf16" if ctx.bf16 else "",
                           att_grad, rte_first=True)
        if not ctx.bf16:
            q.copy_(dq)
        q = kv = dq = dkv = None                                       # bf16: the tables go before dX / dW
        dx, dw, db = _linear_backward(ctx, dproj, x, None, hi, lo, w_cat, ctx.needs_input_grad[0])
        return dx, dw, db, dkvr, None, None, None, None, None, None, None, None, None


class _FoldWeights(torch.autograd.Function):
    """(W_cat, b_cat) of the typed projection: per type  [W_q ; K'_p ; V'_p ...]  (hgt_fold_weights, conv.py:96-104)."""

    @staticmethod
    def forward(ctx, module, plan, lt, *params):
        m = module
        T, R, H, d_in, d = m.num_types, m.num_relations, m.n_heads, m.in_dim, m.out_dim
        dev = params[0].device
        st = _stream()
        tabs = [m._ptrs(n, ts, dev) for n, ts in (("wq", [l.weight for l in m.q_linears]), ("bq", [l.bias for l in m.q_linears]),
                                                 ("wk", [l.weight for l in m.k_linears]), ("bk", [l.bias for l in m.k_linears]),
                                                 ("wv", [l.weight for l in m.v_linears]), ("bv", [l.bias for l in m.v_linears]))]
        w_cat = torch.empty((max(lt.cat_rows, 1), d_in), dtype=torch.float32, device=dev)
        b_cat = torch.empty(max(lt.cat_rows, 1), dtype=torch.float32, device=dev)
        _lib.call("hgt_fold_weights", *[t.data_ptr() for t in tabs], m.relation_att.data_ptr(), m.relation_msg.data_ptr(),
                  m.relation_pri.data_ptr(), T, R, H, d_in, d, plan.n_pairs, plan.pair_type_dev.data_ptr(),
                  plan.pair_rel_dev.data_ptr(), lt.cat_row0_dev.data_ptr(), lt.q_row0_dev.data_ptr(), w_cat.data_ptr(),
                  b_cat.data_ptr(), st)
        ctx.module, ctx.plan, ctx.lt, ctx.tabs = m, plan, lt, tabs
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return w_cat, b_cat

    @staticmethod
    def backward(ctx, dw_cat, db_cat):
        m, plan, lt, tabs = ctx.module, ctx.plan, ctx.lt, ctx.tabs
        T, R, H, d_in, d, dk = m.num_types, m.num_relations, m.n_heads, m.in_dim, m.out_dim, m.d_k
        dev = dw_cat.device
        dw_cat, db_cat = dw_cat.contiguous(), db_cat.contiguous()
        f32 = dict(dtype=torch.float32, device=dev)
        d_wk, d_wv = torch.empty((T, d, d_in), **f32), torch.empty((T, d, d_in), **f32)
        d_bk, d_bv = torch.empty((T, d), **f32), torch.empty((T, d), **f32)
        d_att, d_msg = torch.empty((R, H, dk, dk), **f32), torch.empty((R, H, dk, dk), **f32)
        d_pri = torch.empty((R, H), **f32)
        _lib.call("hgt_fold_backward_det" if ctx.det else "hgt_fold_backward", dw_cat.data_ptr(), db_cat.data_ptr(), tabs[2].data_ptr(), tabs[3].data_ptr(),
                  tabs[4].data_ptr(), tabs[5].data_ptr(), m.relation_att.data_ptr(), m.relation_msg.data_ptr(),
                  m.relation_pri.data_ptr(), T, R, H, d_in, d, plan.n_pairs, plan.pair_type_dev.data_ptr(),
                  plan.pair_rel_dev.data_ptr(), lt.cat_row0_dev.data_ptr(), d_wk.data_ptr(), d_bk.data_ptr(),
                  d_wv.data_ptr(), d_bv.data_ptr(), d_att.data_ptr(), d_msg.data_ptr(), d_pri.data_ptr(), _stream())
        # W_q / b_q rows of W_cat are plain copies: their gradient is the matching slice
        d_wq = [dw_cat[lt.q_row0[t]:lt.q_row0[t] + d] for t in range(T)]
        d_bq = [db_cat[lt.q_row0[t]:lt.q_row0[t] + d] for t in range(T)]
        grads = d_wq + d_bq + list(d_wk.unbind(0)) + list(d_bk.unbind(0)) + list(d_wv.unbind(0)) + list(d_bv.unbind(0))
        return (None, None, None) + tuple(grads) + (d_att, d_msg, d_pri)


class _UpdateEpilogue(torch.autograd.Function):
    """out[perm[k]] = LayerNorm_t(o[k] * sigmoid(skip[t]) + x[k] * (1 - sigmoid(skip[t])))   (conv.py:129-133);
    skip=None: the plain residual o + x of DenseHGTConv (conv.py:261,273).  type_row0: [T+2] int32 row prefix (rows past
    type_row0[T] are written as zeros), perm: rank-order row -> output row, or None.  seed (one int64 on the device) with
    p > 0: `o` is the pre-dropout tensor and the kernels apply the mask of (seed, p) (fused dropout)."""

    @staticmethod
    def forward(ctx, o, x, skip, norm_w, norm_b, type_row0, T, perm, type_active=None, seed=None, p=0.0):
        N, d = o.shape
        o, x = o.contiguous(), x.contiguous()
        # with type_active (sharded training, trimmed layers) the rows past the active prefix of a type have no output
        # row: they are zero (never an uninitialised row a later stage could read) and receive no gradient
        # (hgt_update_backward skips them)
        out = (torch.zeros if type_active is not None else torch.empty)((N, d), dtype=torch.float32, device=o.device)
        args = (o.data_ptr(), x.data_ptr(), type_row0.data_ptr(), T, _lib.ptr(skip), _lib.ptr(norm_w), _lib.ptr(norm_b),
                _lib.ptr(perm), _lib.ptr(type_active), N, d, out.data_ptr(), None, None)
        if seed is not None:
            _lib.call("hgt_update_epilogue_drop", *args, seed.data_ptr(), p, _stream())
        else:
            _lib.call("hgt_update_epilogue", *args, _stream())
        ctx.T, ctx.has_norm, ctx.has_skip, ctx.p = T, norm_w is not None, skip is not None, p
        ctx.det = torch.are_deterministic_algorithms_enabled()
        ctx.save_for_backward(o, x, skip, norm_w, type_row0, perm, type_active, seed)
        return out

    @staticmethod
    def backward(ctx, dout):
        o, x, skip, norm_w, type_row0, perm, type_active, seed = ctx.saved_tensors
        T = ctx.T
        N, d = o.shape
        dev = o.device
        dout = dout.contiguous()
        d_o, d_x = torch.empty_like(o), torch.empty_like(x)
        d_skip = torch.empty(T, dtype=torch.float32, device=dev) if ctx.has_skip else None
        d_nw = torch.empty((T, d), dtype=torch.float32, device=dev) if ctx.has_norm else None
        d_nb = torch.empty((T, d), dtype=torch.float32, device=dev) if ctx.has_norm else None
        args = (dout.data_ptr(), o.data_ptr(), x.data_ptr(), type_row0.data_ptr(), T, _lib.ptr(skip), _lib.ptr(norm_w),
                _lib.ptr(perm), _lib.ptr(type_active), N, d, d_o.data_ptr(), d_x.data_ptr(), _lib.ptr(d_skip),
                _lib.ptr(d_nw), _lib.ptr(d_nb))
        drop = () if seed is None else (seed.data_ptr(), ctx.p)
        sfx = "" if seed is None else "_drop"
        if ctx.det:
            wsb = ctypes.c_size_t()
            _lib.call("hgt_update_backward_det_workspace_bytes", N, T, d, ctypes.byref(wsb))
            ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
            _lib.call("hgt_update_backward%s_det" % sfx, *args, ws.data_ptr(), ws.numel(), *drop, _stream())
        else:
            _lib.call("hgt_update_backward" + sfx, *args, *drop, _stream())
        return d_o, d_x, d_skip, d_nw, d_nb, None, None, None, None, None, None


class _TanhDropout(torch.autograd.Function):
    """out = tanh(x) * mask * s over the first n_rows of x [N, d], the remaining rows unchanged (hgt_tanh_dropout): the GNN
    adapter's tanh and dropout as one pass that keeps `out` alone for the backward."""

    @staticmethod
    def forward(ctx, x, n_rows, seed, p):
        x = x.contiguous()
        N, d = x.shape
        out = torch.empty_like(x)
        _lib.call("hgt_tanh_dropout", x.data_ptr(), n_rows, N, d, seed.data_ptr(), p, out.data_ptr(), _stream())
        ctx.n_rows, ctx.p = n_rows, p
        ctx.save_for_backward(out, seed)
        return out

    @staticmethod
    def backward(ctx, dout):
        out, seed = ctx.saved_tensors
        N, d = out.shape
        dout = dout.contiguous()
        d_x = torch.empty_like(out)
        _lib.call("hgt_tanh_dropout_bwd", dout.data_ptr(), out.data_ptr(), ctx.n_rows, N, d, seed.data_ptr(), ctx.p,
                  d_x.data_ptr(), _stream())
        return d_x, None, None, None


def typed_linear(a, w_cat, b_cat, table, width, out_elems, impl=0, act=0, zero_ranges=(), tables16=None):
    return _TypedLinear.apply(a, w_cat, b_cat, table, width, out_elems, impl, act, tuple(zero_ranges), tables16)


def _proj_layout(plan, lt, d, bf16):
    """(zero_ranges, tables16) of the projection's typed GEMM: the flat [Q | pad | K'V' table | zero row] buffer with its
    padding and zero row cleared, or, with bf16 tables, the fp32 Q buffer and the bf16 [K'|V'] table (zero row cleared)."""
    kv_end = lt.kv_off + plan.kv_rows * 2 * d
    if bf16:
        return (), (lt.q_groups, plan.n_nodes * d, lt.kv_groups, lt.kv_off,
                    ((kv_end - lt.kv_off, lt.proj_elems - lt.kv_off),))
    return ((plan.n_nodes * d, lt.kv_off), (kv_end, lt.proj_elems)), None


def _rte_tables(m, w_cat, plan, lt, bf16):
    """(kvr, kvr16) of a layer: with RTE the table [P*240+1, 2d] (+ all-zero row) and, with bf16 tables, kvr is its
    gradient stand-in and kvr16 the bf16 table; (None, None) without RTE."""
    if not m.use_RTE:
        return None, None
    P, d, d_in = plan.n_pairs, m.out_dim, m.in_dim
    # RT = lin(emb.weight) [240, d_in] (conv.py:299), then projected with every pair's K'/V' weights (no bias)
    rt = typed_linear(m.emb.emb.weight, m.emb.lin.weight, m.emb.lin.bias, lt.rt_group, d_in,
                      _plan.RTE_MAX_LEN * d_in, 1).view(_plan.RTE_MAX_LEN, d_in)
    n_kvr = (P * _plan.RTE_MAX_LEN + 1) * 2 * d
    zero = ((P * _plan.RTE_MAX_LEN * 2 * d, n_kvr),)
    if bf16:
        kvr, _, kvr16 = typed_linear(rt, w_cat, None, lt.rte_groups, d, n_kvr, 1, 0, (),
                                     (None, 0, lt.rte_groups, 0, zero))
        return kvr, kvr16
    return typed_linear(rt, w_cat, None, lt.rte_groups, d, n_kvr, 1, 0, zero), None


def _project(m, x, w_cat, b_cat, plan, lt, bf16, impl):
    """Typed projections of a layer: the flat [Q | pad | K'V' table | zero row] buffer and, with RTE, the RTE table
    [P*240+1, 2d] (+ all-zero row).  bf16: those two are gradient stand-ins and the third result holds what the edge kernel
    reads, (Q, bf16 [K'|V'] table, bf16 RTE table or None); otherwise it is None.  impl: the projection GEMM's (gemm_impl;
    the RTE tables stay fp32 SIMT)."""
    zero_ranges, tables16 = _proj_layout(plan, lt, m.out_dim, bf16)
    res = typed_linear(x, w_cat, b_cat, lt.proj_groups, m.out_dim, lt.proj_elems, impl, 0, zero_ranges, tables16)
    proj, q, kv = res if bf16 else (res, None, None)
    kvr, kvr16 = _rte_tables(m, w_cat, plan, lt, bf16)
    return proj, kvr, ((q, kv, kvr16) if bf16 else None)


# layers that ran a training forward: GraphedTrainStep freezes their recompute_tables switch at capture
_TRAINED_LAYERS = weakref.WeakSet()


def recompute_switches(params):
    """{layer: bool(recompute_tables)} of the layers that ran a training forward and own one of `params`."""
    owned = {id(p) for p in params}
    return {m: bool(m.recompute_tables) for m in list(_TRAINED_LAYERS) if any(id(p) in owned for p in m.parameters())}


# modules with a dropout site (layers, GNN) that ran a training forward: GraphedTrainStep freezes their fused_dropout
_DROPOUT_MODULES = weakref.WeakSet()


def fused_dropout_switches(params):
    """{module: bool(fused_dropout)} of the layers / GNNs that ran a training forward and own one of `params`."""
    owned = {id(p) for p in params}
    return {m: bool(m.fused_dropout) for m in list(_DROPOUT_MODULES) if any(id(p) in owned for p in m.parameters())}


def _project_edge(m, x, w_cat, b_cat, plan, lt, impl, want_att):
    """Typed projections and edge attention of a layer: (agg, att).  m.recompute_tables, read here once per training
    forward, selects _ProjectEdgeLean (the backward rebuilds the projection tables); otherwise the projection buffer is
    kept for the backward (_project + _EdgeAttention)."""
    d, H = m.out_dim, m.n_heads
    bf16 = bf16_tables()
    if torch.is_grad_enabled():
        _TRAINED_LAYERS.add(m)
        _DROPOUT_MODULES.add(m)
        if m.recompute_tables:
            kvr, kvr16 = _rte_tables(m, w_cat, plan, lt, bf16)
            return _ProjectEdgeLean.apply(x, w_cat, b_cat, kvr, plan, lt, d, H, want_att, m.edge_variant, impl, bf16,
                                          kvr16)
    proj, kvr, tables16 = _project(m, x, w_cat, b_cat, plan, lt, bf16, impl)
    return _EdgeAttention.apply(proj, kvr, plan, lt, d, H, want_att, m.edge_variant, tables16)


def hgt_conv_autograd(m, node_inp, node_type, edge_index, edge_type, edge_time, active=None, kv_runs=None, plan=None,
                      want_att=None):
    """`active` (sharded training, trimmed layers): active[t] = number of leading nodes of type t (rank order) that are
    destinations here; Q / a_linear / update run for them only, the remaining rows (halo sources) only get K'/V' rows and
    their output rows stay zero.  `kv_runs`: per-pair row ranges that need K'/V' (plan.layer_tables).  `plan`: an explicit
    plan (a trimmed layer's view, trim.py) instead of the cached plan of the tensors.  `want_att`: materialise m.att
    (default m.keep_att)."""
    d_in, d, H, T, R = m.in_dim, m.out_dim, m.n_heads, m.num_types, m.num_relations
    if plan is None:
        plan = _plan.get_plan(node_type, edge_index, edge_type, edge_time if m.use_RTE else None, T, R)
    if want_att is None:
        want_att = bool(m.keep_att)
    N, P = plan.n_nodes, plan.n_pairs
    if node_inp.shape[0] != N:
        raise ValueError("node_inp has %d rows but node_type has %d" % (node_inp.shape[0], N))
    x = node_inp if plan.sorted_types else node_inp.index_select(0, plan.perm.long())
    if active is not None and not plan.sorted_types:
        raise ValueError("`active` needs a type-sorted node order")
    lt = _plan.layer_tables(plan, d_in, d, active, kv_runs)

    # 1. relation matrices folded into the typed K/V weights; typed projections -> flat [Q | pad | K'V' table | zero row]
    params = ([l.weight for l in m.q_linears] + [l.bias for l in m.q_linears] +
              [l.weight for l in m.k_linears] + [l.bias for l in m.k_linears] +
              [l.weight for l in m.v_linears] + [l.bias for l in m.v_linears] +
              [m.relation_att, m.relation_msg, m.relation_pri])
    w_cat, b_cat = _FoldWeights.apply(m, plan, lt, *params)
    impl = gemm_impl(m.linear_impl, bf16_matmuls())

    # 2. fused edge kernel (with m.recompute_tables one stage with the projection, whose backward rebuilds the tables)
    agg, att = _project_edge(m, x, w_cat, b_cat, plan, lt, impl, want_att)
    _set_att(m, att)

    # 3. a_linears on gelu(agg) (conv.py:119,125): the gelu is applied inside the operand split / the dX epilogue
    wa_cat = torch.cat([l.weight for l in m.a_linears], 0)
    ba_cat = torch.cat([l.bias for l in m.a_linears], 0)
    o = typed_linear(agg, wa_cat, ba_cat, lt.upd_groups, d, N * d, impl, 1).view(N, d)
    p_fused = fused_drop_p(m)                                                    # conv.py:125, inside the update kernels
    if m.training and m.drop.p > 0 and not p_fused:
        o = m.drop(o)                                                            # conv.py:125

    # 4. gated skip + LayerNorm, written in original node order; rows of unknown type stay zero (conv.py:120)
    norm_w = torch.stack([n.weight for n in m.norms]) if m.use_norm else None
    norm_b = torch.stack([n.bias for n in m.norms]) if m.use_norm else None
    return _UpdateEpilogue.apply(o, x, m.skip, norm_w, norm_b, plan.type_row0_dev, T,
                                 None if plan.sorted_types else plan.perm, lt.type_active_dev,
                                 drop_seed(o.device) if p_fused else None, p_fused)


def dense_hgt_forward(m, node_inp, node_type, edge_index, edge_type, edge_time):
    """DenseHGTConv.forward (conv.py:143-280): the same message() => the same projection / edge kernels, then
        y   = LayerNorm_t(drop(a_linear_t(agg)) + x)                     conv.py:261-266   (no gelu, no skip gate)
        out = out_norm(drop(out_linear(gelu(mid_linear(y)))) + y)        conv.py:273-274   (FFN shared by all types)
    built from the same differentiable stages: typed GEMMs (the gelu of the FFN sits in the operand split of out_linear
    and in the dX epilogue of its backward) and the residual mode of the update epilogue.  Used for inference and
    training alike (under no_grad the stages simply do not record)."""
    d_in, d, H, T, R = m.in_dim, m.out_dim, m.n_heads, m.num_types, m.num_relations
    plan = _plan.get_plan(node_type, edge_index, edge_type, edge_time if m.use_RTE else None, T, R)
    N, P = plan.n_nodes, plan.n_pairs
    if node_inp.shape[0] != N:
        raise ValueError("node_inp has %d rows but node_type has %d" % (node_inp.shape[0], N))
    dev = node_inp.device
    x = node_inp if plan.sorted_types else node_inp.index_select(0, plan.perm.long())
    lt = _plan.layer_tables(plan, d_in, d)
    params = ([l.weight for l in m.q_linears] + [l.bias for l in m.q_linears] +
              [l.weight for l in m.k_linears] + [l.bias for l in m.k_linears] +
              [l.weight for l in m.v_linears] + [l.bias for l in m.v_linears] +
              [m.relation_att, m.relation_msg, m.relation_pri])
    w_cat, b_cat = _FoldWeights.apply(m, plan, lt, *params)
    impl = gemm_impl(m.linear_impl, bf16_matmuls())
    agg, att = _project_edge(m, x, w_cat, b_cat, plan, lt, impl, bool(m.keep_att))
    _set_att(m, att)

    p_fused = fused_drop_p(m)
    drop = m.training and m.drop.p > 0 and not p_fused
    wa_cat = torch.cat([l.weight for l in m.a_linears], 0)
    ba_cat = torch.cat([l.bias for l in m.a_linears], 0)
    o = typed_linear(agg, wa_cat, ba_cat, lt.upd_groups, d, N * d, impl, 0).view(N, d)              # conv.py:261
    if drop:
        o = m.drop(o)
    norm_w = torch.stack([n.weight for n in m.norms]) if m.use_norm else None
    norm_b = torch.stack([n.bias for n in m.norms]) if m.use_norm else None
    y = _UpdateEpilogue.apply(o, x, None, norm_w, norm_b, plan.type_row0_dev, T, None, None,
                              drop_seed(dev) if p_fused else None, p_fused)                        # rank order

    n_known = plan.type_row0[T]
    key = ("dense_ffn", d)
    tabs = plan._layer_tables.get(key)
    if tabs is None:
        one = lambda w_: _plan._pack_groups([(0, n_known, 0, 1, 0, 1)], [(0, w_)], dev)            # noqa: E731
        tabs = plan._layer_tables[key] = (one(2 * d), one(d),
                                          _plan._to_dev_async(np.asarray([0, n_known, N], dtype=np.int32), dev))
    hmid = typed_linear(y, m.mid_linear.weight, m.mid_linear.bias, tabs[0], 2 * d, N * 2 * d, impl, 0,
                        ((n_known * 2 * d, N * 2 * d),)).view(N, 2 * d)
    z = typed_linear(hmid, m.out_linear.weight, m.out_linear.bias, tabs[1], d, N * d, impl, 1,
                     ((n_known * d, N * d),)).view(N, d)                                             # gelu inside
    if drop:
        z = m.drop(z)
    # shared out_norm over every known row, residual with y, written in original node order; unknown types -> zeros
    return _UpdateEpilogue.apply(z, y, None, m.out_norm.weight.view(1, d), m.out_norm.bias.view(1, d), tabs[2], 1,
                                 None if plan.sorted_types else plan.perm, None,
                                 drop_seed(dev) if p_fused else None, p_fused)
