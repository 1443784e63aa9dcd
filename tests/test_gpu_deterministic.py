"""Deterministic training backward under torch.use_deterministic_algorithms(True) (run on an H100: ``pytest -m gpu``).

With the flag on, every autograd stage of the training path calls the atomic-free backward kernels: the destination
pass + source-major row passes of the edge backward, hgt_typed_linear_bwd_det, hgt_update_backward_det and
hgt_fold_backward_det.  Two training steps from identical module state and inputs must then give bitwise equal outputs
and gradients, and those gradients must still match float64 autograd within the bounds of test_gpu_grad_parity.py.
With the flag off the default kernels run, and none of the deterministic entry points is called.
"""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, plan as P                                           # noqa: E402
from tests.test_gpu_grad_parity import (CASES, FRO_BOUND, _case, _compare_all, _dev, _f64_params, _graph,  # noqa: E402
                                        _layer, _native_layer, _oracle_layer)

DET_ENTRY_POINTS = {"hgt_plan_source_index", "hgt_edge_backward_det_workspace_bytes", "hgt_edge_backward_dst",
                    "hgt_edge_backward_rows", "hgt_typed_linear_bwd_det_workspace_bytes", "hgt_typed_linear_bwd_det",
                    "hgt_update_backward_det_workspace_bytes", "hgt_update_backward_det", "hgt_fold_backward_det"}
DEFAULT_BWD_ENTRY_POINTS = {"hgt_edge_backward", "hgt_typed_linear_bwd", "hgt_update_backward", "hgt_fold_backward"}


@contextlib.contextmanager
def _deterministic(on, warn_only=False):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _assert_bitwise(a, b, tag):
    (o1, dx1, g1), (o2, dx2, g2) = a, b
    assert torch.equal(o1, o2), "%s: out differs between two identical steps" % tag
    assert torch.equal(dx1, dx2), "%s: d node_inp differs between two identical steps" % tag
    assert set(g1) == set(g2)
    bad = [k for k in sorted(g1) if not ((g1[k] is None and g2[k] is None) or torch.equal(g1[k], g2[k]))]
    assert not bad, "%s: gradients differ between two identical steps: %s" % (tag, bad)


def _hgt_step(state, ctor_args, impl, x, g, w, dev):
    import pyhgt_b200
    m = pyhgt_b200.HGTConv(*ctor_args)
    m.load_state_dict(state)
    m = m.to(dev).train()
    m.linear_impl = impl
    return _native_layer(m, x, g, w, dev)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_deterministic_step_repeats_bitwise_and_matches_float64(name, impl, monkeypatch):
    """Every grad-parity case x linear_impl 0 / 1: two steps with the flag on are bitwise equal, and the result is
    within FRO_BOUND of float64 autograd."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, state, x, w, ref = _case(name)
    d, H, T, R, rte, _ = CASES[name]
    args = (d, d, T, R, H, 0.0, True, rte)
    with _deterministic(True):
        a = _hgt_step(state, args, impl, x, g, w, dev)
        b = _hgt_step(state, args, impl, x, g, w, dev)
    _assert_bitwise(a, b, "%s impl %d" % (name, impl))
    _compare_all("deterministic %s impl %d" % (name, impl), a, ref, FRO_BOUND[name])


def _split_rows_graph(seed):
    """Unsorted types, RTE, edges that match no triple, and one source that sends 2,600 edges with one relation and one
    time gap: its K'/V' row and its <pair, dt> RTE row both lie above TILE_SPLIT_EDGES (split rows of the row passes),
    next to the two split destinations of _graph."""
    T, R = 3, 4
    g = _graph(T, R, seed, False)
    gen = torch.Generator().manual_seed(seed + 7)
    cand = [int(i) for i in (g.node_type == 0).nonzero().flatten() if int(i) % 11]
    src = cand[3]
    n = 2600
    dst = torch.randint(0, g.num_nodes, (n,), generator=gen)
    g.edge_index = torch.cat([g.edge_index, torch.stack([torch.full((n,), src, dtype=torch.int64), dst])], 1)
    g.edge_type = torch.cat([g.edge_type, torch.zeros(n, dtype=torch.int64)])
    g.edge_time = torch.cat([g.edge_time, torch.full((n,), 7, dtype=torch.int64)])
    g.edge_type[::7] = R + 5                                     # unmatched: relation out of range
    g.node_type[::11] = T + 2                                    # unmatched: node type out of range (src is kept)
    unknown = g.node_type >= T
    ok = ~(unknown[g.edge_index[0]] | unknown[g.edge_index[1]] | (g.edge_type >= R))
    shared = ok & (g.edge_index[0] == src) & (g.edge_type == 0) & (g.edge_time == 7)
    assert int(shared.sum()) > P.TILE_SPLIT_EDGES and int((~ok).sum()) > 1000
    return g, T, R


@pytest.mark.parametrize("impl", [0, 1])
def test_split_source_and_rte_rows_repeat_bitwise_and_match_float64(impl, monkeypatch):
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, T, R = _split_rows_graph(95)
    d, H = 256, 8
    m = _layer(d, H, T, R, True, 96)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(97))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(98))
    params = _f64_params(m)
    xr = x.double().requires_grad_(True)
    out = _oracle_layer(params, xr, g, m)
    (out * w.double()).sum().backward()
    ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
    state = m.state_dict()
    args = (d, d, T, R, H, 0.0, True, True)
    with _deterministic(True):
        a = _hgt_step(state, args, impl, x, g, w, dev)
        b = _hgt_step(state, args, impl, x, g, w, dev)
    _assert_bitwise(a, b, "split rows impl %d" % impl)
    _compare_all("deterministic split rows impl %d" % impl, a, ref, (3e-5, 3e-4))


def test_three_layer_gnn_and_dense_hgt_repeat_bitwise():
    """A 3-layer GNN (typed adapter + HGT layers with RTE) and a DenseHGTConv step (FFN, residual epilogue)."""
    import pyhgt_b200
    from pyhgt_b200.model import GNN
    dev = _dev()
    old_keep = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = False
    try:
        T, R = 3, 4
        g = _graph(T, R, 101, False)
        nt, ei, et, tm = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev)
        x = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(102)).to(dev)
        w = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(103)).to(dev)
        torch.manual_seed(104)
        gnn = GNN(64, 128, T, R, 4, 3, 0.0, "hgt", True, True, True)
        dense = pyhgt_b200.DenseHGTConv(128, 128, T, R, 4, 0.0, True, True)
        x2 = torch.randn(g.num_nodes, 128, generator=torch.Generator().manual_seed(105)).to(dev)

        def gnn_step():
            m = GNN(64, 128, T, R, 4, 3, 0.0, "hgt", True, True, True)
            m.load_state_dict(gnn.state_dict())
            m = m.to(dev).train()
            xg = x.clone().requires_grad_(True)
            o = m(xg, nt, tm, ei, et)
            (o * w).sum().backward()
            return o.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}

        def dense_step():
            m = pyhgt_b200.DenseHGTConv(128, 128, T, R, 4, 0.0, True, True)
            m.load_state_dict(dense.state_dict())
            m = m.to(dev).train()
            xg = x2.clone().requires_grad_(True)
            o = m(xg, nt, ei, et, tm)
            (o * w).sum().backward()
            return o.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}

        with _deterministic(True):
            _assert_bitwise(gnn_step(), gnn_step(), "3-layer GNN")
            _assert_bitwise(dense_step(), dense_step(), "DenseHGTConv")
    finally:
        pyhgt_b200.HGTConv.keep_att = old_keep


@pytest.mark.parametrize("flag", [False, True])
def test_inference_out_and_att_repeat_bitwise(flag):
    """Inference owns every output row / tile and merges hub pieces in piece order: deterministic with the flag off too."""
    import pyhgt_b200
    dev = _dev()
    T, R = 3, 4
    g = _graph(T, R, 111, False)
    m = _layer(256, 8, T, R, True, 112).to(dev).eval()
    m.keep_att = True
    x = torch.randn(g.num_nodes, 256, generator=torch.Generator().manual_seed(113)).to(dev)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    runs = []
    with _deterministic(flag), torch.no_grad():
        for _ in range(2):
            P.clear_plan_cache()
            out = m(x, *args)
            runs.append((out.clone(), m.att.clone()))
    assert isinstance(m, pyhgt_b200.HGTConv)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_deterministic_step_on_sync_free_batch_has_no_host_sync():
    """A to_torch(prebuild_plan=True) batch (sync-free plan): the deterministic step, including the first build of the
    source-major index on the new plan, runs under torch's sync debug mode "error"."""
    import pyhgt_b200
    from pyhgt_b200 import data as hdata
    from tests.conftest import load_golden
    from tests.test_data_ingest import _GraphStub
    dev = _dev()
    fx = load_golden("to_torch")
    g = _GraphStub(fx["types"], fx["meta_graph"])
    T = len(fx["types"])
    d = fx["node_feature"].shape[1]

    def batch():
        # edge_time stays referenced: the prebuilt plan is cached under all four tensors
        nf, nt, etime, ei, et, node_dict, edge_dict = hdata.to_torch(fx["feature"], fx["time"], fx["edge_list"], g,
                                                                    device=dev, prebuild_plan=True)
        return nf, nt, etime, ei, et, len(edge_dict)

    nf, nt, etime, ei, et, R = batch()
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, T, R, 1, 0.0, True, False).to(dev).train()
    m.keep_att = False

    def step(nf, nt, ei, et):
        m.zero_grad(set_to_none=True)
        xg = nf.clone().requires_grad_(True)
        m(xg, nt, ei, et).square().sum().backward()
        return xg.grad, {k: p.grad for k, p in m.named_parameters()}

    with _deterministic(True):
        ref = step(nf, nt, ei, et)                                 # warm-up (library load, workspace sizes)
        torch.cuda.synchronize()
        P.clear_plan_cache()
        nf2, nt2, etime2, ei2, et2, _ = batch()
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = step(nf2, nt2, ei2, et2)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(ref[0], got[0])
    assert all(torch.equal(ref[1][k], got[1][k]) for k in ref[1] if ref[1][k] is not None)


@pytest.mark.parametrize("mode", ["off", "on", "warn_only"])
def test_flag_selects_the_backward_entry_points(mode, monkeypatch):
    """Flag off: the default kernels only, none of the deterministic entry points.  Flag on (warn_only included): the
    deterministic twins only."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    called = []
    real_call = _lib.call

    def spy(name, *args):
        called.append(name)
        return real_call(name, *args)

    monkeypatch.setattr(_lib, "call", spy)
    g, state, x, w, _ = _case("h3_d96_rte")
    d, H, T, R, rte, _ = CASES["h3_d96_rte"]
    with _deterministic(mode != "off", warn_only=mode == "warn_only"):
        _hgt_step(state, (d, d, T, R, H, 0.0, True, rte), 0, x, g, w, dev)
    names = set(called)
    if mode == "off":
        assert not names & DET_ENTRY_POINTS, sorted(names & DET_ENTRY_POINTS)
        assert DEFAULT_BWD_ENTRY_POINTS <= names
    else:
        assert {"hgt_edge_backward_dst", "hgt_edge_backward_rows", "hgt_typed_linear_bwd_det", "hgt_update_backward_det",
                "hgt_fold_backward_det"} <= names
        assert not names & DEFAULT_BWD_ENTRY_POINTS, sorted(names & DEFAULT_BWD_ENTRY_POINTS)
