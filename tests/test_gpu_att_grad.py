"""Gradient of HGTConv.att (run on an H100: ``pytest -m gpu``).

In the reference, att = softmax(res_att, edge_index_i) (pyHGT/conv.py:108) is a node of the autograd graph, so a loss
term on it reaches every parameter and node_inp.  Here a loss that reads att takes hgt_edge_att_grad_prep and the *_att
edge backward calls (csrc/edge_bwd.cu, ATT = true); a loss that does not read it runs exactly the calls without it.

  * every <VEC, NCH> instance of the three ATT passes, fp32 and bf16 tables, RTE off and on, a hub destination in every
    graph, "hot" scores, atomic and deterministic: dq, d[K'|V'] and d RTE against float64 autograd of
    sum(agg * dagg) + sum(att * datt) on the same (widened) tables (the shapes and helpers of test_gpu_edge_instances);
  * zero datt gives bitwise the gradients of the path without att, and an att left out of the loss launches the same
    kernels as a forward that never made it;
  * the reference's own gradients of sum(out * w) + sum(att * w_att) (tests/golden/att_*.pt, scripts/make_att_golden.py);
  * bitwise repeatable under torch.use_deterministic_algorithms, inside GraphedTrainStep, and pickling after a
    training forward.
"""
import contextlib
import copy
import difflib
import io
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pyhgt_b200 import _lib, graphed, plan as P, synth
from tests.test_gpu_edge_instances import (CASES, DTYPES, _check_hot, _dev, _edge_ref, _forward, _graph, _max_err,
                                           _plan, _q_scale, _st, _tables)


@contextlib.contextmanager
def _deterministic(on):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@contextlib.contextmanager
def _keep_att(on):
    import pyhgt_b200
    old = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = on
    try:
        yield
    finally:
        pyhgt_b200.HGTConv.keep_att = old


def _edge_backward(plan, q, kv, kvr, agg, dagg, stats, d, H, det, dtype, datt=None, att=None):
    """dq, d[K'|V'], d RTE of one edge backward: the calls without att (datt None) or prep + the *_att calls."""
    from pyhgt_b200.autograd import _att_grad_prep, _edge_backward_det
    dev = q.device
    N = plan.n_nodes
    sfx = "_bf16" if dtype == "bf16" else ""
    rte = kvr is not None
    dq = torch.empty(N, d, device=dev)
    dkv = torch.empty(plan.kv_rows + 1, 2 * d, device=dev)
    dkvr = torch.empty_like(kvr, dtype=torch.float32) if rte else None
    att_grad = _att_grad_prep(att, datt, plan, H) if datt is not None else None
    if det:
        _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, sfx, att_grad)
    else:
        fn, extra = "hgt_edge_backward", ()
        if att_grad is not None:
            fn, extra = "hgt_edge_backward_att", (att_grad[0].data_ptr(), att_grad[1].data_ptr())
        ws = torch.empty(256, dtype=torch.uint8, device=dev)
        _lib.call(fn + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(), dagg.data_ptr(),
                  stats.data_ptr(), *extra, plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
                  plan.rte_row.data_ptr() if rte else None, plan.tiles.data_ptr(), plan.n_tiles, N, d, H,
                  plan.kv_rows + 1, kvr.shape[0] if rte else 0, dq.data_ptr(), dkv.data_ptr(), _lib.ptr(dkvr),
                  ws.data_ptr(), ws.numel(), _lib.ptr(plan.tile_counts_dev), _st())
    torch.cuda.synchronize()
    return dq, dkv, dkvr


# ---------------------------------------------------------------------------------------------------------------------
# 1. every kernel instance against float64

def test_att_shape_list_reaches_every_instance():
    """CASES (shared with test_gpu_edge_instances) reaches all 12 <VEC, NCH> lane maps, with RTE off and on and hot."""
    from tests.test_gpu_edge_instances import lane_map
    every = {(v, n) for v in (1, 2, 4) for n in (1, 2, 4, 8)}
    for rte in (False, True):
        assert {lane_map(d, H) for d, H, r, hot in CASES if r == rte and not hot} == every
    assert {lane_map(d, H) for d, H, _, hot in CASES if hot} == every


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d,H,rte,hot", CASES)
def test_att_backward_matches_fp64(d, H, rte, hot, det, dtype):
    """prep + hgt_edge_backward[_dst/_rows]_att[_bf16] against float64 autograd of sum(agg*dagg) + sum(att*datt); the
    deterministic path repeats bitwise."""
    dev = _dev()
    plan, T = _plan(d, H, rte, seed=3 * d + H)
    q, kv, kvr = _tables(plan, d, rte, d + 2, DTYPES[dtype], _q_scale(d, H, hot))
    N, E = plan.n_nodes, plan.n_edges
    att = torch.empty(E, H, device=dev)
    agg, stats = _forward(plan, T, q, kv, kvr, d, H, 0, att, dtype)
    gen = torch.Generator().manual_seed(6)
    dagg = torch.randn(N, d, generator=gen).to(dev)
    datt = torch.randn(E, H, generator=gen).to(dev)
    got = _edge_backward(plan, q, kv, kvr, agg, dagg, stats, d, H, det, dtype, datt, att)

    q64 = q.cpu().double().requires_grad_(True)
    kv64 = kv.cpu().double().requires_grad_(True)
    kvr64 = kvr.cpu().double().requires_grad_(True) if rte else None
    ref_agg, att_ref, _, _ = _edge_ref(plan, q64, kv64, kvr64, H)
    if hot:
        _check_hot(att_ref.detach())
    eid = plan.csr_eid[:E].cpu().long()
    ((ref_agg * dagg.cpu().double()).sum() + (att_ref * datt.cpu().double()[eid]).sum()).backward()
    rows = plan.kv_rows
    errs = [_max_err(got[0].cpu(), q64.grad), _max_err(got[1][:rows].cpu(), kv64.grad[:rows])]
    if rte:
        errs.append(_max_err(got[2][:-1].cpu(), kvr64.grad[:-1]))
    assert max(errs) <= 5e-5, "max errors (dq, dkv[, dkvr]): %s" % ", ".join("%.3g" % e for e in errs)
    if det:
        again = _edge_backward(plan, q, kv, kvr, agg, dagg, stats, d, H, det, dtype, datt, att)
        for a, b in zip(got, again):
            if a is not None:
                assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d,H", [(40, 8), (64, 4), (100, 4), (256, 8), (512, 8)])
def test_att_prep_writes_csr_order_and_c(d, H, dtype):
    """hgt_edge_att_grad_prep: datt_csr[c] = datt[csr_eid[c]] exactly, C_i = sum_e att_e datt_e (hub included), and the
    same bits on a second call."""
    from pyhgt_b200.autograd import _att_grad_prep
    dev = _dev()
    plan, T = _plan(d, H, True, seed=d)
    q, kv, kvr = _tables(plan, d, True, d, DTYPES[dtype])
    E = plan.n_edges
    att = torch.empty(E, H, device=dev)
    _forward(plan, T, q, kv, kvr, d, H, 0, att, dtype)
    datt = torch.randn(E, H, generator=torch.Generator().manual_seed(2)).to(dev)
    datt_csr, c = _att_grad_prep(att, datt, plan, H)
    datt_csr2, c2 = _att_grad_prep(att, datt, plan, H)
    torch.cuda.synchronize()
    eid = plan.csr_eid[:E].long()
    assert torch.equal(datt_csr[:E], datt[eid])
    rp = plan.row_ptr.cpu().long()
    dst = torch.repeat_interleave(torch.arange(plan.n_nodes), rp[1:] - rp[:-1])
    ref = torch.zeros(plan.n_nodes, H, dtype=torch.float64).index_add_(0, dst, (att[eid] * datt[eid]).cpu().double())
    has_in = (rp[1:] - rp[:-1]) > 0
    torch.testing.assert_close(c.cpu().double()[has_in], ref[has_in], rtol=1e-5, atol=1e-5)
    assert torch.equal(c[has_in.to(dev)], c2[has_in.to(dev)]) and torch.equal(datt_csr, datt_csr2)


# ---------------------------------------------------------------------------------------------------------------------
# 2. zero datt: bitwise the path without att

def _unique_rows_plan(seed):
    """One type, one relation, every source sends one edge (each [K'|V'] row has one contribution) and no destination
    above the split threshold: the atomic backward then has a fixed result, so two of its runs can be compared bitwise."""
    dev = _dev()
    gen = torch.Generator().manual_seed(seed)
    n_src, n_dst = 3000, 250
    src = torch.randperm(n_src, generator=gen)
    dst = torch.randint(0, n_dst, (n_src,), generator=gen)
    nt = torch.zeros(n_src, dtype=torch.int64)
    ei = torch.stack([src, dst])
    et = torch.zeros(n_src, dtype=torch.int64)
    plan = P.build_plan(nt.to(dev), ei.to(dev), et.to(dev), None, 1, 1)
    assert plan.n_split == 0
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d,H", [(40, 8), (64, 4), (100, 4), (256, 8), (512, 8)])
def test_zero_datt_is_bitwise_the_path_without_att(d, H, det, dtype):
    """datt = 0 through the ATT calls gives bitwise the gradients of the calls without att: ds = p((dp + 0) - (D + 0)).
    The atomic path runs on a graph whose rows take one contribution each (its float reductions have a fixed result
    there); the deterministic path on the hub graph with RTE."""
    dev = _dev()
    if det:
        plan, T = _plan(d, H, True, seed=d + 7)
        rte = True
    else:
        plan, T, rte = _unique_rows_plan(d), 1, False
    q, kv, kvr = _tables(plan, d, rte, d + 3, DTYPES[dtype])
    E = plan.n_edges
    att = torch.empty(E, H, device=dev)
    agg, stats = _forward(plan, T, q, kv, kvr, d, H, 0, att, dtype)
    dagg = torch.randn(plan.n_nodes, d, generator=torch.Generator().manual_seed(8)).to(dev)
    base = _edge_backward(plan, q, kv, kvr, agg, dagg, stats, d, H, det, dtype)
    zero = _edge_backward(plan, q, kv, kvr, agg, dagg, stats, d, H, det, dtype, torch.zeros(E, H, device=dev), att)
    for a, b in zip(base, zero):
        if a is not None:
            assert torch.equal(a, b)


def _layer(d, H, T, R, rte, seed, dense=False):
    import pyhgt_b200
    torch.manual_seed(seed)
    cls = pyhgt_b200.DenseHGTConv if dense else pyhgt_b200.HGTConv
    m = cls(d, d, T, R, H, 0.0, True, rte)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "skip" in name or "relation_pri" in name or "norm" in name:
                p.add_(0.3 * torch.randn(p.shape))
    return m


def _module_step(m, x, g, w, w_att, att_scale, dev):
    """One training step of a layer: loss = sum(out * w) + att_scale * sum(att * w_att) (att_scale None: no att term).
    Returns (out, d node_inp, {name: grad})."""
    xg = x.to(dev).requires_grad_(True)
    out = m(xg, g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    loss = (out * w.to(dev)).sum()
    if att_scale is not None:
        assert m.att.requires_grad
        loss = loss + att_scale * (m.att * w_att.to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    return out.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_zero_att_term_is_bitwise_the_step_without_it(dense):
    """Module level, deterministic backward: sum(out*w) + 0*sum(att) and sum(out*w) give bitwise equal gradients.
    The atomic backward is not compared here: its float reductions (edge backward, dW, update) add in an order that
    varies from run to run, so two of its steps are not bitwise equal even on the same path.  Its zero-datt identity is
    checked at kernel level instead (test_zero_datt_is_bitwise_the_path_without_att), on a graph where every row takes
    one contribution."""
    dev = _dev()
    T, R, d, H = 3, 2, 64, 4
    g = _graph(T, R, seed=31)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(2))
    w_att = torch.randn(g.num_edges, H, generator=torch.Generator().manual_seed(3))
    m = _layer(d, H, T, R, True, 5, dense)
    with _keep_att(True), _deterministic(True):
        a = _module_step(copy.deepcopy(m).to(dev).train(), x, g, w, w_att, 0.0, dev)
        b = _module_step(copy.deepcopy(m).to(dev).train(), x, g, w, w_att, None, dev)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]:
        assert torch.equal(a[2][k], b[2][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_unused_att_launches_the_same_backward_kernels(det, monkeypatch):
    """keep_att on with a loss that does not read att: the same C-ABI calls (forward and backward) and the same
    backward kernel launch list (CUPTI, in order) as keep_att off.  The forward's lists differ by design: under the
    deterministic flag torch fills the uninitialised att buffer.  Both lists come from a warm profiler: one profiled
    step runs first, so a first CUPTI session in the process is never one of the two compared.  A session can still
    miss its first kernel record (seen on an H100 as a missing leading fill of the backward, keep_att off in both
    sessions), so each session first runs spin kernels, which the backward never launches, and the list is the kernels
    after the last one recorded."""
    from torch.profiler import profile, ProfilerActivity
    import pyhgt_b200
    dev = _dev()
    T, R, d, H = 3, 2, 128, 8
    g = _graph(T, R, seed=32)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(2))
    m = _layer(d, H, T, R, True, 6).to(dev).train()
    calls = []
    real_call = _lib.call

    def spy(name, *args):
        calls.append(name)
        return real_call(name, *args)
    monkeypatch.setattr(_lib, "call", spy)

    args = [t.to(dev) for t in (g.node_type, g.edge_index, g.edge_type, g.edge_time)]
    wd = w.to(dev)

    def step(keep):
        with _keep_att(keep), _deterministic(det):
            m.zero_grad(set_to_none=True)
            (m(x.to(dev).requires_grad_(True), *args) * wd).sum().backward()     # warm-up: plan, source index
            m.zero_grad(set_to_none=True)
            calls.clear()
            loss = (m(x.to(dev).requires_grad_(True), *args) * wd).sum()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    torch.cuda._sleep(1000)
                    torch.cuda.synchronize()
                loss.backward()
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            marks = [i for i, n in enumerate(names) if "spin_kernel" in n]
            assert marks, names[:4]
            return list(calls), names[marks[-1] + 1:], (m.att is not None) and m.att.requires_grad
    step(False)                                                            # warms the profiler
    calls_on, kernels_on, att_grad = step(True)
    calls_off, kernels_off, _ = step(False)
    assert att_grad
    assert not any("_att" in c for c in calls_on), calls_on
    assert calls_on == calls_off, "\n".join(difflib.unified_diff(calls_off, calls_on, "keep_att off", "on", lineterm=""))
    assert any("k_edge_bwd" in k for k in kernels_on)
    assert kernels_on == kernels_off, "\n".join(difflib.unified_diff(kernels_off, kernels_on, "keep_att off", "on",
                                                                     lineterm=""))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the reference's own gradients

def _check_grad(got, ref, what):
    got, ref = got.float().cpu(), ref.float()
    scale = ref.abs().max().item()
    fro = ((got - ref).norm() / ref.norm().clamp_min(1e-30)).item()
    assert torch.allclose(got, ref, rtol=1e-3, atol=1e-3 * max(scale, 1e-6)), \
        "%s: max abs err %.3g (scale %.3g, rel fro %.3g)" % (what, (got - ref).abs().max().item(), scale, fro)
    assert fro <= 2e-3, "%s: relative Frobenius error %.3g" % (what, fro)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("name", ["att_rte", "att_norte", "att_only", "att_dense"])
def test_att_loss_matches_reference_gradients(name, det):
    """sum(out * w) + sum(att * w_att) (att_only: the att term alone) through HGTConv / DenseHGTConv against the
    reference's autograd on the same module (hub destination, RTE on and off)."""
    import pyhgt_b200
    from tests.conftest import load_golden
    dev = _dev()
    fx = load_golden(name)
    c = fx["cfg"]
    cls = pyhgt_b200.DenseHGTConv if c["dense"] else pyhgt_b200.HGTConv
    m = cls(c["in_dim"], c["out_dim"], c["num_types"], c["num_relations"], c["n_heads"], 0.2, c["use_norm"],
            c["use_RTE"])
    m.load_state_dict(fx["state_dict"], strict=True)
    m = m.to(dev).eval()
    x = fx["node_inp"].to(dev).requires_grad_(True)
    with _keep_att(True), _deterministic(det):
        out = m(x, fx["node_type"].to(dev), fx["edge_index"].to(dev), fx["edge_type"].to(dev),
                fx["edge_time"].to(dev))
        assert m.att.requires_grad
        _check_grad(m.att.detach(), fx["att"], name + " att")
        loss = (m.att * fx["grad_att_weight"].to(dev)).sum()
        if fx["grad_weight"] is not None:
            loss = loss + (out * fx["grad_weight"].to(dev)).sum()
        loss.backward()
    _check_grad(x.grad, fx["grad_node_inp"], name + " d node_inp")
    got = {k: p.grad for k, p in m.named_parameters()}
    for k, ref in fx["grad_params"].items():
        assert got[k] is not None, "no gradient for " + k
        _check_grad(got[k], ref, name + " d " + k)


# ---------------------------------------------------------------------------------------------------------------------
# 4. determinism, graphed steps, pickling

def _gnn(T, R, f_in, n_hid, seed):
    from pyhgt_b200.model import GNN
    torch.manual_seed(seed)
    return GNN(f_in, n_hid, T, R, 4, 2, 0.0, "hgt", True, True, True)


def _att_term(gnn, weights, n_edges=None):
    return sum((gc.base_conv.att[:n_edges] * w).sum() for gc, w in zip(gnn.gcs, weights))


@pytest.mark.gpu
def test_two_layer_gnn_with_att_terms_repeats_bitwise():
    """Deterministic flag: two identical steps of a 2-layer GNN whose loss reads every layer's att give bitwise equal
    gradients, and the att terms change them."""
    dev = _dev()
    T, R = 3, 2
    g = _graph(T, R, seed=33)
    x = torch.randn(g.num_nodes, 48, generator=torch.Generator().manual_seed(1)).to(dev)
    w = torch.randn(g.num_nodes, 64, generator=torch.Generator().manual_seed(2)).to(dev)
    w_att = [torch.randn(g.num_edges, 4, generator=torch.Generator().manual_seed(3 + l)).to(dev) for l in range(2)]
    base = _gnn(T, R, 48, 64, 7)
    args = [t.to(dev) for t in (g.node_type, g.edge_time, g.edge_index, g.edge_type)]

    def step(with_att):
        gnn = copy.deepcopy(base).to(dev).train()
        h = gnn(x, *args)
        loss = (h * w).sum() + (_att_term(gnn, w_att) if with_att else 0.0)
        loss.backward()
        torch.cuda.synchronize()
        return {k: p.grad.clone() for k, p in gnn.named_parameters()}
    with _keep_att(True), _deterministic(True):
        a, b, plain = step(True), step(True), step(False)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    moved = [k for k in a if not torch.equal(a[k], plain[k])]
    assert any(k.startswith("gcs.0.") for k in moved) and any(k.startswith("adapt_ws") for k in moved)


T_G, R_G, F_IN, N_HID, N_CLS = 3, 4, 48, 64, 5


def _batches(seeds):
    return [synth.make_random(n, e, T_G, R_G, seed=s, sorted_types=True, self_loops=20)
            for n, e, s in zip((400, 310, 455, 380), (3000, 2200, 3400, 2900), seeds)]


def _features(b):
    return torch.randn(b.num_nodes, F_IN, generator=torch.Generator().manual_seed(7 + b.num_nodes))


def _labels(b):
    n0 = int((b.node_type == 0).sum())
    return torch.randint(0, N_CLS, (n0,), generator=torch.Generator().manual_seed(b.num_nodes))


def _att_loss_fn(gnn, head, rows, pad_node, w_att):
    """Task loss + 0.5 * sum over the layers of att * w_att on the real edges: padding edges are self loops on the last
    (padding) node, graphed.pad_batch."""
    def loss_fn(x, nt, tm, ei, et, targets):
        h = gnn(x, nt, tm, ei, et)[:rows]
        real = (ei[1] != pad_node).to(torch.float32)[:, None]
        att = sum((gc.base_conv.att * real * w).sum() for gc, w in zip(gnn.gcs, w_att))
        return F.nll_loss(F.log_softmax(head(h), -1), targets[0], ignore_index=-100) + 0.5 * att
    return loss_fn


@pytest.mark.gpu
@pytest.mark.parametrize("det", [True, False])
def test_graphed_recipe_with_att_loss_matches_eager_steps(det):
    """GraphedTrainStep (AdamW, OneCycleLR, clip 1.0) with a loss that reads each layer's att over the real edges
    matches the same eager steps; bitwise under the deterministic flag."""
    dev = _dev()
    batches = _batches((1, 2, 3, 4)) + _batches((5, 6))
    counts = [max(int((b.node_type == t).sum()) for b in batches) + 5 for t in range(T_G)]
    pairs = {(int(b.node_type[s_]), int(r_)) for b in batches
             for s_, r_ in zip(b.edge_index[0].tolist(), b.edge_type.tolist())}
    sig = graphed.GraphSignature(counts, max(b.edge_type.numel() for b in batches) + 100, pairs, R_G, F_IN)
    torch.manual_seed(11)
    from pyhgt_b200.model import GNN
    gnn = GNN(F_IN, N_HID, T_G, R_G, 4, 2, 0.0, "hgt", True, True, True).to(dev).train()
    head = torch.nn.Linear(N_HID, N_CLS).to(dev)
    gnn2, head2 = copy.deepcopy(gnn), copy.deepcopy(head)
    w_att = [torch.randn(sig.n_edges, 4, generator=torch.Generator().manual_seed(20 + l)).to(dev) for l in range(2)]
    p1 = list(gnn.parameters()) + list(head.parameters())
    p2 = list(gnn2.parameters()) + list(head2.parameters())

    def recipe(params):
        opt = torch.optim.AdamW(params, lr=torch.tensor(5e-4, device=dev), capturable=True)
        sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-3, total_steps=40, pct_start=0.1,
                                                    anneal_strategy="linear", final_div_factor=10,
                                                    cycle_momentum=False)
        return opt, sched
    opt1, sched1 = recipe(p1)
    opt2, sched2 = recipe(p2)
    pad_node = sig.n_nodes - 1
    with _keep_att(True):
        step = graphed.GraphedTrainStep(_att_loss_fn(gnn, head, sig.type_counts[0], pad_node, w_att), sig, dev,
                                        optimizer=opt1, clip_norm=1.0, targets={0: ((), torch.int64, -100)})
        eager_loss = _att_loss_fn(gnn2, head2, sig.type_counts[0], pad_node, w_att)
        with _deterministic(det):
            for b in batches:
                x, y = _features(b), _labels(b)
                with warnings.catch_warnings(record=True) as caught:
                    warnings.simplefilter("always")
                    step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
                # the first call captures: the layers' .att of its eager steps must not carry their AccumulateGrad
                # nodes (made on the default stream) into the capture
                assert not [w_ for w_ in caught if "AccumulateGrad" in str(w_.message)]
                sched1.step()
                px, pnt, ptm, pei, pet, _ = graphed.pad_batch(sig, x, b.node_type, b.edge_time, b.edge_index,
                                                              b.edge_type)
                assert (pei[1, :b.edge_type.numel()] != pad_node).all() and (pei[1, b.edge_type.numel():] == pad_node).all()
                tens = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (px, pnt, ptm, pei, pet)]
                tgt = torch.full((sig.type_counts[0],), -100, dtype=torch.int64)
                tgt[:y.numel()] = y
                P.rebuild_plan(tens[1], tens[3], tens[4], tens[2], T_G, R_G, sig.host_meta())
                opt2.zero_grad()
                eager_loss(*tens, {0: tgt.to(dev)}).backward()
                assert gnn2.gcs[0].base_conv.att.requires_grad
                torch.nn.utils.clip_grad_norm_(p2, 1.0, foreach=True)
                opt2.step()
                sched2.step()
    torch.cuda.synchronize()
    for a, b in zip(p1, p2):
        if det:
            assert torch.equal(a, b), "parameters differ after the steps"
        else:
            rel = (a.double() - b.double()).norm().item() / max(b.double().norm().item(), 1e-30)
            assert rel < 1e-5, rel


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_deepcopy_and_save_after_training_forward(dense):
    """copy.deepcopy and torch.save right after a training forward with keep_att on: the copy's att is a detached
    tensor with the same values, and the layer's own att still carries its gradient."""
    dev = _dev()
    T, R, d, H = 3, 2, 64, 4
    g = synth.make_random(300, 2000, T, R, seed=9, self_loops=10)
    m = _layer(d, H, T, R, True, 8, dense).to(dev).train()
    x = torch.randn(g.num_nodes, d, device=dev, requires_grad=True)
    with _keep_att(True):
        out = m(x, g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
        assert m.att.requires_grad and m.att.grad_fn is not None
        c = copy.deepcopy(m)
        buf = io.BytesIO()
        torch.save(m, buf)
        buf.seek(0)
        loaded = torch.load(buf, weights_only=False)
    for other in (c, loaded):
        assert not other.att.requires_grad and other.att.grad_fn is None
        assert torch.equal(other.att, m.att.detach())
    (out.sum() + m.att.sum()).backward()
    assert x.grad is not None


@pytest.mark.gpu
@pytest.mark.parametrize("rte", [False, True])
def test_source_index_carries_csr_positions_from_the_same_sort(rte):
    """source_index(..., with_pos=True): the same ptr / dst / oth as the index without positions, and pos[j] is a CSR
    position whose key, destination and other-table row are those of entry j, every position once."""
    plan, _ = _plan(64, 4, rte, seed=12)
    E = plan.n_edges
    whiches = ["kv", "rte"] if rte else ["kv"]
    plain = {w: P.source_index(plan, w) for w in whiches}
    for w in whiches:
        idx = P.source_index(plan, w, with_pos=True)
        assert idx is not plain[w] and plain[w].pos is None and P.source_index(plan, w) is idx
        for name in ("ptr", "dst", "oth"):
            a, b = getattr(plain[w], name), getattr(idx, name)
            assert (a is None and b is None) or torch.equal(a[:E] if name != "ptr" else a, b[:E] if name != "ptr" else b)
        pos = idx.pos[:E].long()
        assert torch.equal(pos.sort().values, torch.arange(E, device=pos.device))
        key, other = (plan.kv_row, plan.rte_row) if w == "kv" else (plan.rte_row, plan.kv_row)
        k = key[:E].long()[pos]
        assert bool((k[1:] >= k[:-1]).all())
        dst = torch.searchsorted(plan.row_ptr.long(), pos, right=True) - 1
        assert torch.equal(dst, idx.dst[:E].long())
        if other is not None:
            assert torch.equal(other[:E][pos], idx.oth[:E])


@pytest.mark.gpu
def test_release_att_graphs_keeps_other_models_att():
    """release_att_graphs(params) detaches the att of the layers owning those parameters only: another model's att
    keeps its graph, and a loss term on it still reaches that model's parameters."""
    from pyhgt_b200.autograd import release_att_graphs
    dev = _dev()
    T, R, d, H = 3, 2, 64, 4
    g = synth.make_random(300, 2000, T, R, seed=10, self_loops=10)
    args = [t.to(dev) for t in (g.node_type, g.edge_index, g.edge_type, g.edge_time)]
    a = _layer(d, H, T, R, True, 1).to(dev).train()
    b = _layer(d, H, T, R, True, 2).to(dev).train()
    x = torch.randn(g.num_nodes, d, device=dev)
    with _keep_att(True):
        a(x, *args)
        b(x, *args)
    release_att_graphs(list(a.parameters()))
    assert not a.att.requires_grad and b.att.requires_grad
    b.att.sum().backward()
    assert b.relation_att.grad is not None and b.relation_att.grad.abs().max() > 0
