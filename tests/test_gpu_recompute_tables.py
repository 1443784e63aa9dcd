"""HGTConv.recompute_tables: the training forward keeps neither Q nor the [K'|V'] table; the backward rebuilds them with
the forward's projection GEMM and runs the source-major edge passes, the [K'|V'] pass writing each row's gradient over
the row itself (run on an H100: ``pytest -m gpu``).

With the deterministic flag on, lean and keep steps must agree bit for bit (outputs, att and every gradient); with it off
the keep path's atomic edge backward differs in rounding only.  The in-place row pass is checked against a separate
gradient buffer on every lane-map instance, with split rows and RTE tables present.
"""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

import pyhgt_b200                                                                      # noqa: E402
from pyhgt_b200 import graphed, plan as P, sharded, synth                              # noqa: E402
from tests.test_gpu_edge_instances import (SHAPES, _edge_ref, _forward, _graph as _edge_graph, _max_err,  # noqa: E402
                                           _tables)
from tests.test_gpu_grad_parity import _graph, _layer                                  # noqa: E402


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@contextlib.contextmanager
def _det(on):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _set_lean(model, on):
    for mod in model.modules():
        if isinstance(mod, pyhgt_b200.HGTConv):
            mod.recompute_tables = on


def _step(model, x, args, w, lean, w_att=None, **kw):
    """One forward + backward: (out, [att of every layer], d x, {parameter: grad})."""
    _set_lean(model, lean)
    model.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    out = model(xg, *args, **kw)
    loss = (out * w).sum()
    convs = [mod for mod in model.modules() if isinstance(mod, pyhgt_b200.HGTConv)]
    if w_att is not None:
        loss = loss + sum((c.att * w_att[:c.att.shape[0]]).sum() for c in convs)
    loss.backward()
    atts = [None if c.att is None else c.att.detach().clone() for c in convs]
    return (out.detach().clone(), atts, xg.grad.clone(),
            {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})


def _assert_bitwise(keep, lean, tag):
    assert torch.equal(keep[0], lean[0]), "%s: output" % tag
    assert len(keep[1]) == len(lean[1])
    for a, b in zip(keep[1], lean[1]):
        assert (a is None and b is None) or torch.equal(a, b), "%s: att" % tag
    assert torch.equal(keep[2], lean[2]), "%s: d node_inp" % tag
    assert set(keep[3]) == set(lean[3]), tag
    bad = [k for k in sorted(keep[3]) if not torch.equal(keep[3][k], lean[3][k])]
    assert not bad, "%s: gradients differ: %s" % (tag, bad)


def _rel(a, b):
    return (a.double() - b.double()).norm().item() / max(b.double().norm().item(), 1e-30)


def _args(g, dev, rte):
    return (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev) if rte else None)


def _keep_then_lean(model, x, args, w, **kw):
    return _step(model, x, args, w, False, **kw), _step(model, x, args, w, True, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the layers: lean == keep bit for bit under the deterministic flag

@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("rte", [False, True])
@pytest.mark.parametrize("d,H", [(64, 4), (256, 8), (400, 8)])
def test_hgtconv_lean_step_is_bitwise_the_keep_step(d, H, rte, norm):
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 31 + d, False)
    torch.manual_seed(d + H)
    m = pyhgt_b200.HGTConv(d, d, T, R, H, 0.0, norm, rte).to(dev).train()
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(2)).to(dev)
    with _det(True):
        keep, lean = _keep_then_lean(m, x, _args(g, dev, rte), w)
    assert keep[1][0] is not None                                      # keep_att: att is compared too
    _assert_bitwise(keep, lean, "d=%d H=%d rte=%s norm=%s" % (d, H, rte, norm))


@pytest.mark.parametrize("rte", [False, True])
def test_simt_projection_and_att_loss_term(rte):
    """linear_impl 1 (fp32 SIMT projection: fp32 x is saved instead of its split) and a loss term on att (the *_att
    passes; the in-place pass reads datt at the entries' CSR positions)."""
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 41, False)
    m = _layer(64, 4, T, R, rte, 5).to(dev).train()
    w = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(2)).to(dev)
    x = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    w_att = torch.randn(g.num_edges, 4, generator=torch.Generator().manual_seed(3)).to(dev)
    with _det(True):
        for impl in (1, 0):
            m.linear_impl = impl
            keep, lean = _keep_then_lean(m, x, _args(g, dev, rte), w, w_att=w_att)
            _assert_bitwise(keep, lean, "impl %d with an att term" % impl)


def test_dense_hgt_and_two_layer_gnn():
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 51, False)
    nt, ei, et, tm = _args(g, dev, True)
    w = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(2)).to(dev)
    torch.manual_seed(7)
    dense = pyhgt_b200.DenseHGTConv(128, 128, T, R, 4, 0.0, True, True).to(dev).train()
    gnn = GNN(64, 128, T, R, 4, 2, 0.0, "hgt", True, True, True).to(dev).train()
    w_att = torch.randn(g.num_edges, 4, generator=torch.Generator().manual_seed(3)).to(dev)
    with _det(True):
        x = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(1)).to(dev)
        _assert_bitwise(*_keep_then_lean(dense, x, (nt, ei, et, tm), w), "DenseHGTConv")
        x = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(1)).to(dev)
        _assert_bitwise(*_keep_then_lean(gnn, x, (nt, tm, ei, et), w), "2-layer GNN")
        _assert_bitwise(*_keep_then_lean(gnn, x, (nt, tm, ei, et), w, w_att=w_att), "2-layer GNN, att terms")


@pytest.mark.parametrize("mode", ["bf16_autocast", "medium"])
@pytest.mark.parametrize("rte", [False, True])
def test_bf16_tables_and_medium_precision(mode, rte):
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 61, False)
    m = _layer(128, 8, T, R, rte, 9).to(dev).train()
    x = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(2)).to(dev)
    w_att = torch.randn(g.num_edges, 8, generator=torch.Generator().manual_seed(3)).to(dev)
    prec = torch.get_float32_matmul_precision()
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "bf16_autocast" else contextlib.nullcontext()
    try:
        if mode == "medium":
            torch.set_float32_matmul_precision("medium")
        with _det(True), ctx:
            _assert_bitwise(*_keep_then_lean(m, x, _args(g, dev, rte), w), mode)
            _assert_bitwise(*_keep_then_lean(m, x, _args(g, dev, rte), w, w_att=w_att), mode + " with an att term")
    finally:
        torch.set_float32_matmul_precision(prec)


@pytest.mark.parametrize("tsig", [False, True])
def test_trimmed_training(tsig):
    """GNN.forward(..., out_nodes=) with and without a TrimSignature: the layers run on trimmed plan views."""
    from pyhgt_b200 import trim
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R, L = 3, 4, 3
    g = _graph(T, R, 71, False)
    nt, ei, et, tm = _args(g, dev, True)
    torch.manual_seed(3)
    gnn = GNN(32, 64, T, R, 4, L, 0.0, "hgt", True, True, True).to(dev).train()
    out_nodes = torch.randperm(g.num_nodes, generator=torch.Generator().manual_seed(4))[:40].to(dev)
    x = torch.randn(g.num_nodes, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.randn(40, 64, generator=torch.Generator().manual_seed(2)).to(dev)
    kw = dict(out_nodes=out_nodes)
    if tsig:
        counts = trim.build_layout(nt, ei, et, tm, out_nodes, T, R, L).counts
        kw["trim_signature"] = trim.TrimSignature(counts + 3, L)
    with _det(True):
        keep, lean = _keep_then_lean(gnn, x, (nt, tm, ei, et), w, **kw)
    _assert_bitwise(keep, lean, "trimmed, tsig=%s" % tsig)


def test_sharded_forward_train_one_rank_and_compacted_tables():
    """ShardedGraph.forward_train with one rank, and the layer on rank 1 of 3's local graph with its active prefixes
    and compacted K'/V' runs (groups that overlap in rows: the projection backward's sub-tables)."""
    from pyhgt_b200.autograd import hgt_conv_autograd
    dev = _dev()
    g = synth.make_random(6000, 60000, 3, 2, seed=12, isolated_frac=0.1, self_loops=100)
    torch.manual_seed(4)
    m = pyhgt_b200.HGTConv(64, 64, 3, 2, 4, 0.0, True, True).to(dev).train()
    x = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(5))
    with _det(True):
        sh = sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, 3, 2, 0, 1, dev)
        w = torch.randn(sh.n_owned, 64, generator=torch.Generator().manual_seed(6)).to(dev)

        class _One(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.conv = m

            def forward(self, x_own):
                return sh.forward_train(self.conv, x_own)

        _assert_bitwise(*_keep_then_lean(_One(), x[sh.owned_global].to(dev), (), w), "forward_train, one rank")

        sh3 = sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, 3, 2, 1, 3, dev)
        assert sh3.kv_runs is not None
        xl = x[sh3.local_global].to(dev)
        w3 = torch.randn(sh3.n_owned, 64, generator=torch.Generator().manual_seed(7)).to(dev)

        class _Local(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.conv = m

            def forward(self, x_local):
                out = hgt_conv_autograd(self.conv, x_local, sh3.node_type, sh3.edge_index, sh3.edge_type, sh3.edge_time,
                                        active=sh3.active_per_type, kv_runs=sh3.kv_runs)
                return out.index_select(0, sh3.own_rows)

        _assert_bitwise(*_keep_then_lean(_Local(), xl, (), w3), "rank 1 of 3, compacted K'/V' runs")


# ---------------------------------------------------------------------------------------------------------------------
# 2. flag off: the keep path's atomic edge backward differs from the source-major passes in rounding only

def test_flag_off_gradients_match_keep():
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 81, False)
    nt, ei, et, tm = _args(g, dev, True)
    torch.manual_seed(8)
    gnn = GNN(64, 256, T, R, 8, 2, 0.0, "hgt", True, True, True).to(dev).train()
    x = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.randn(g.num_nodes, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    with _det(False):
        keep, lean = _keep_then_lean(gnn, x, (nt, tm, ei, et), w)
    assert torch.equal(keep[0], lean[0])                               # the forward is the same either way
    # fp32 sums in another order: on an H100 the largest difference here was 1.1e-6 (d node_inp), and 2.2e-6 on the c4
    # step (scripts/recompute_train_bench.py)
    assert _rel(lean[2], keep[2]) < 5e-6
    for k in keep[3]:
        assert _rel(lean[3][k], keep[3][k]) < 5e-6, (k, _rel(lean[3][k], keep[3][k]))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the in-place row pass: hgt_edge_backward_rows[_att] with grad == own

def _split_rows_plan(rte, seed):
    """The edge-instance graph (a split destination) plus 2,600 edges from one source with one relation and one time:
    its K'/V' row and its RTE row are split rows of the row passes."""
    dev = _dev()
    T, R = 3, 2
    g = _edge_graph(T, R, seed=seed)
    n_extra, src = 2600, 17
    gen = torch.Generator().manual_seed(seed + 5)
    g.edge_index = torch.cat([g.edge_index, torch.stack([torch.full((n_extra,), src, dtype=torch.int64),
                                                         torch.randint(0, g.num_nodes, (n_extra,), generator=gen)])], 1)
    g.edge_type = torch.cat([g.edge_type, torch.zeros(n_extra, dtype=torch.int64)])
    g.edge_time = torch.cat([g.edge_time, torch.full((n_extra,), 7, dtype=torch.int64)])
    plan = P.build_plan(g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev),
                        g.edge_time.to(dev) if rte else None, T, R)
    return plan, T


@pytest.mark.parametrize("att", [False, True])
@pytest.mark.parametrize("rte", [False, True])
@pytest.mark.parametrize("d,H", SHAPES)
def test_in_place_row_pass_matches_separate_grad_and_float64(d, H, rte, att):
    from pyhgt_b200.autograd import _att_grad_prep, _edge_backward_det
    dev = _dev()
    plan, T = _split_rows_plan(rte, seed=d + 3 * H)
    q, kv, kvr = _tables(plan, d, rte, d + 1, torch.float32)
    N, E = plan.n_nodes, plan.n_edges
    att_t = torch.empty(E, H, device=dev)
    agg, stats = _forward(plan, T, q, kv, kvr, d, H, 0, att_t)
    gen = torch.Generator().manual_seed(9)
    dagg = torch.randn(N, d, generator=gen).to(dev)
    datt = torch.randn(E, H, generator=gen).to(dev) if att else None
    att_grad = _att_grad_prep(att_t, datt, plan, H) if att else None

    dq, dkv = torch.empty(N * d, device=dev), torch.empty_like(kv)
    dkvr = torch.empty_like(kvr) if rte else None
    _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, "", att_grad)
    own = kv.clone()
    dq2 = torch.empty(N * d, device=dev)
    dkvr2 = torch.empty_like(kvr) if rte else None
    _edge_backward_det(q, own, kvr, agg, dagg, stats, plan, d, H, dq2, own, dkvr2, "", att_grad, rte_first=True)
    torch.cuda.synchronize()
    for which in (["kv", "rte"] if rte else ["kv"]):                   # split rows really are present
        assert int(P.source_index(plan, which, att).counts_dev[1]) > 0, which
    assert torch.equal(own, dkv)
    assert torch.equal(dq2, dq)
    if rte:
        assert torch.equal(dkvr2, dkvr)

    q64 = q.cpu().double().requires_grad_(True)
    kv64 = kv.cpu().double().requires_grad_(True)
    kvr64 = kvr.cpu().double().requires_grad_(True) if rte else None
    ref_agg, att_ref, _, _ = _edge_ref(plan, q64, kv64, kvr64, H)
    loss = (ref_agg * dagg.cpu().double()).sum()
    if att:
        loss = loss + (att_ref * datt.cpu().double()[plan.csr_eid[:E].cpu().long()]).sum()
    loss.backward()
    rows = plan.kv_rows
    errs = [_max_err(dq2.view(N, d).cpu(), q64.grad), _max_err(own[:rows].cpu(), kv64.grad[:rows])]
    if rte:
        errs.append(_max_err(dkvr2[:-1].cpu(), kvr64.grad[:-1]))
    assert max(errs) <= 5e-5, "max errors (dq, dkv[, dkvr]): %s" % ", ".join("%.3g" % e for e in errs)
    assert not own[rows:].any()                                        # the trailing all-zero row's gradient


# ---------------------------------------------------------------------------------------------------------------------
# 4. memory: the c4 stack (3 layers, d = 256, 8 heads, no RTE) on a reduced ogbn-mag-shaped graph

def test_lean_step_peak_memory_is_below_keep():
    dev = _dev()
    L, D, H = 3, 256, 8
    g = synth.make_mag_shaped(0.05)
    nt, ei, et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([pyhgt_b200.HGTConv(D, D, g.num_types, g.num_relations, H, 0.0, True, False)
                                  for _ in range(L)]).to(dev).train()
    for mod in layers:
        mod.keep_att = False
    x = torch.randn(g.num_nodes, D, generator=torch.Generator().manual_seed(0)).to(dev)
    w = torch.randn(g.num_nodes, D, generator=torch.Generator().manual_seed(1)).to(dev)

    def peak(lean):
        _set_lean(layers, lean)
        layers.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        h = x
        for mod in layers:
            h = mod(h, nt, ei, et)
        (h * w).sum().backward()
        del h
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated(dev) - base

    for lean in (False, True):                                         # warm-up: plans, source index, tables
        peak(lean)
    keep, lean = peak(False), peak(True)
    lt = P.layer_tables(P.get_plan(nt, ei, et, None, g.num_types, g.num_relations), D, D)
    # keep peaks in the last layer's edge backward: L saved buffers and dproj.  Lean peaks in that layer's projection
    # backward: the recomputed buffer (now dproj), the GEMM's bf16 hi/lo split of it (as large) and dX [N, d].  The gap
    # is (L - 1) buffers less one dX; one more [N, d] of slack covers workspaces (measured on an H100: 0.853 GB here,
    # against 0.965 - 0.099 GB)
    need = (L - 1) * lt.proj_elems * 4 - 2 * g.num_nodes * D * 4
    assert keep - lean >= need, "keep %.3f GB, lean %.3f GB, need a gap of %.3f GB" % (keep / 1e9, lean / 1e9, need / 1e9)


# ---------------------------------------------------------------------------------------------------------------------
# 5. graph capture

def test_graphed_train_step_replays_the_eager_lean_step(monkeypatch):
    from tests.test_gpu_graphed_train import _batches, _features, _labels, _loss_fn, _model, _signature
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    dev = _dev()
    batches = _batches()
    sig = _signature(batches)
    gnn, head = _model("hgt", dropout=0.0)
    _set_lean(gnn, True)
    params = list(gnn.parameters()) + list(head.parameters())
    step = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev, params=params,
                                    targets={0: ((), torch.int64, -100)})
    with _det(True):
        for b in batches:
            x, y = _features(b), _labels(b)
            loss, = step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
            torch.cuda.synchronize()
            g_loss = loss.clone()
            static = [p.grad for p in params]
            g_grads = [gr.clone() for gr in static]
            for p in params:
                p.grad = None
            step._rebuild_plan()
            ref = step.loss_fn(step.x, step.nt, step.tm, step.ei, step.et, step.y)
            ref.backward()
            assert torch.equal(g_loss, ref.detach())
            for p, gr in zip(params, g_grads):
                assert torch.equal(gr, p.grad), "replayed lean gradient differs from the eager lean step"
            for p, gr in zip(params, static):
                p.grad = gr
        gnn.gcs[0].base_conv.recompute_tables = False
        with pytest.raises(RuntimeError, match="recompute_tables"):
            b = batches[0]
            step(_features(b), b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: _labels(b)})
