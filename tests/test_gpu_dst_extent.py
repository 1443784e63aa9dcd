"""Inference over each type's destination extent: an HGTConv inference forward computes Q, the edge pass and the a_linear
only for the rows of each type up to its last destination (plan.GraphPlan.dst_extent); the rows past it have no in-edges
and take the a_linear bias in the update epilogue.  The output must be bitwise the output of the same module on the same
plan with the extents forced to the full type counts (the tables every row used to get)."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pyhgt_b200 import HGTConv, graphed, plan as P, synth          # noqa: E402
from pyhgt_b200.model import GNN                                  # noqa: E402

T, R, D, H = 3, 2, 64, 4


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _graph(counts, blocks, unmatched=(), shuffle=False, seed=0):
    """blocks: (source type, destination type, edges, fraction of the destination type's rows that receive them);
    unmatched: (destination type, edges) whose relation is R, i.e. matches no <source type, relation> pair."""
    g = torch.Generator().manual_seed(seed)
    starts = np.concatenate([[0], np.cumsum(counts)]).tolist()
    node_type = torch.cat([torch.full((c,), t, dtype=torch.int64) for t, c in enumerate(counts)])
    src, dst, rel = [], [], []
    for r, (s, t, m, frac) in enumerate(list(blocks) + [(0, t, m, 1.0) for t, m in unmatched]):
        src.append(torch.randint(0, counts[s], (m,), generator=g) + starts[s])
        dst.append(torch.randint(0, max(1, int(counts[t] * frac)), (m,), generator=g) + starts[t])
        rel.append(torch.full((m,), r % R if r < len(blocks) else R, dtype=torch.int64))
    src = torch.cat(src) if src else torch.zeros(0, dtype=torch.int64)
    dst = torch.cat(dst) if dst else torch.zeros(0, dtype=torch.int64)
    rel = torch.cat(rel) if rel else torch.zeros(0, dtype=torch.int64)
    if shuffle:
        p = torch.randperm(node_type.numel(), generator=g)
        nt = torch.empty_like(node_type)
        nt[p] = node_type
        node_type, src, dst = nt, p[src], p[dst]
    etime = torch.randint(0, 240, (src.numel(),), generator=g)
    return synth.HeteroGraph(node_type, torch.stack([src, dst]), rel, etime, T, R, "dst-extent")


COUNTS = [300, 500, 200]
GRAPHS = {
    "no_in_edges_first": lambda: _graph(COUNTS, [(0, 1, 3000, 1.0), (1, 2, 2000, 1.0)]),
    "no_in_edges_middle": lambda: _graph(COUNTS, [(1, 0, 3000, 1.0), (1, 2, 2000, 1.0)]),
    "no_in_edges_last": lambda: _graph(COUNTS, [(2, 0, 3000, 1.0), (2, 1, 2000, 1.0)]),
    "trailing_tails": lambda: _graph(COUNTS, [(1, 0, 3000, 0.5), (0, 1, 2000, 0.3), (0, 2, 900, 0.7)]),
    "no_edges": lambda: _graph(COUNTS, []),
    "unmatched_only": lambda: _graph(COUNTS, [(1, 0, 3000, 0.6)], unmatched=[(2, 400)]),
    "unsorted_types": lambda: _graph(COUNTS, [(1, 0, 3000, 0.5), (0, 2, 900, 1.0)], shuffle=True),
}


class _Inputs:
    def __init__(self, g, dev, seed=0):
        self.g = g
        self.nt, self.ei, self.et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)
        self.tm = g.edge_time.to(dev)
        self.x = torch.randn(g.num_nodes, D, generator=torch.Generator().manual_seed(seed)).to(dev)

    def plan(self, rte):
        return P.get_plan(self.nt, self.ei, self.et, self.tm if rte else None, T, R)


def _module(norm=True, rte=False, dropout=0.2, seed=0):
    torch.manual_seed(seed)
    m = HGTConv(D, D, T, R, H, dropout, norm, rte).to(_dev()).eval()
    with torch.no_grad():
        m.skip.uniform_(-1.0, 1.0)
        for lin in m.a_linears:
            lin.bias.uniform_(-0.5, 0.5)
        for n in m.norms:
            n.weight.uniform_(0.5, 1.5)
            n.bias.uniform_(-0.2, 0.2)
    return m


@contextlib.contextmanager
def _full_extents(plan):
    """The same plan with dst_extent = type counts: the tables and update epilogue of every row."""
    saved = plan.dst_extent
    plan.dst_extent = list(plan.type_count[:plan.num_types])
    try:
        yield
    finally:
        plan.dst_extent = saved


@contextlib.contextmanager
def _per_stage(on):
    saved = HGTConv.event_sink
    HGTConv.event_sink = [] if on else None
    try:
        yield
    finally:
        HGTConv.event_sink = saved


def _both(plan, fn):
    a = fn()
    with _full_extents(plan):
        b = fn()
    torch.cuda.synchronize()
    return a, b


def _assert_equal(a, b, what="output"):
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        if x is None:
            assert y is None
            continue
        assert torch.isfinite(x).all(), what
        assert torch.equal(x, y), "%s differs from the full-extent tables: max |diff| %.3g" % (
            what, (x - y).abs().max().item())


def _numpy_extent(g):
    nt = g.node_type.numpy()
    deg = np.bincount(g.edge_index[1].numpy(), minlength=nt.size)
    order = np.argsort(np.where((nt >= 0) & (nt < T), nt, T), kind="stable")     # rank order
    ext = []
    for t in range(T):
        rows = order[nt[order] == t]
        hit = np.nonzero(deg[rows] > 0)[0]
        ext.append(int(hit[-1]) + 1 if hit.size else 0)
    return ext


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_plan_extent_matches_numpy(name):
    g = GRAPHS[name]()
    inp = _Inputs(g, _dev())
    plan = inp.plan(False)
    assert plan.dst_extent == _numpy_extent(g)
    assert all(0 <= e <= c for e, c in zip(plan.dst_extent, plan.type_count))


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("norm,rte", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("per_stage", [False, True])
def test_extent_forward_is_bitwise_the_full_forward(name, norm, rte, per_stage):
    inp = _Inputs(GRAPHS[name](), _dev())
    m = _module(norm, rte)
    plan = inp.plan(rte)
    lt = P.layer_tables(plan, D, D, dst=True)
    assert (lt.type_dst_dev is not None) == (plan.dst_extent != plan.type_count[:T])
    if name != "unsorted_types":
        assert lt.type_dst_dev is not None, "the graph should have rows past an extent"

    def run():
        m.keep_att = True
        with torch.no_grad(), _per_stage(per_stage):
            out = m(inp.x, inp.nt, inp.ei, inp.et, inp.tm if rte else None)
        return out, m.att
    _assert_equal(*_both(plan, run))


@pytest.mark.parametrize("mode", ["autocast_bf16", "matmul_medium"])
@pytest.mark.parametrize("per_stage", [False, True])
def test_extent_forward_bitwise_under_reduced_precision(mode, per_stage):
    inp = _Inputs(GRAPHS["trailing_tails"](), _dev())
    m = _module(True, True)
    plan = inp.plan(True)

    def run():
        old = torch.get_float32_matmul_precision()
        ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "autocast_bf16" else contextlib.nullcontext()
        if mode == "matmul_medium":
            torch.set_float32_matmul_precision("medium")
        try:
            with torch.no_grad(), ctx, _per_stage(per_stage):
                return m(inp.x, inp.nt, inp.ei, inp.et, inp.tm)
        finally:
            torch.set_float32_matmul_precision(old)
    _assert_equal(*_both(plan, run))


@pytest.mark.parametrize("layers", [2, 3])
@pytest.mark.parametrize("name", ["no_in_edges_first", "trailing_tails", "unsorted_types"])
def test_gnn_stack_with_emit_split(layers, name):
    inp = _Inputs(GRAPHS[name](), _dev())
    torch.manual_seed(1)
    gnn = GNN(D, D, T, R, H, layers, dropout=0.2, prev_norm=True, last_norm=True, use_RTE=True).to(_dev()).eval()
    assert all(gc.base_conv.emit_split for gc in gnn.gcs[:-1])
    plan = inp.plan(True)

    def run():
        with torch.no_grad():
            return gnn(inp.x, inp.nt, inp.tm, inp.ei, inp.et)
    _assert_equal(*_both(plan, run))


def test_graphed_forward_replay_matches_eager_extent_forward():
    dev = _dev()
    batches = [_graph(COUNTS, [(1, 0, 2000 + 100 * s, 0.5), (0, 2, 700, 1.0)], seed=s) for s in (1, 2)]
    sig = graphed.GraphSignature([c + 7 for c in COUNTS], 3000, [(1, 0), (0, 1)], R, D)
    m = _module(True, True)
    fwd = graphed.GraphedForward(lambda x, nt, tm, ei, et: m(x, nt, ei, et, tm), sig, dev)
    for b in batches:
        x = torch.randn(b.num_nodes, D, generator=torch.Generator().manual_seed(3))
        fwd(x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
        torch.cuda.synchronize()
        graph_out = fwd.out.clone()
        # eager on the padded inputs: new tensors, so a synchronous plan with extents
        args = [t.clone() for t in (fwd.x, fwd.nt, fwd.tm, fwd.ei, fwd.et)]
        plan = P.get_plan(args[1], args[3], args[4], args[2], T, R)
        assert plan.dst_extent != plan.type_count[:T]
        with torch.no_grad():
            eager = m(args[0], args[1], args[3], args[4], args[2])
        torch.cuda.synchronize()
        _assert_equal(eager, graph_out, "graph replay vs eager extent forward")


def test_sync_free_plans_keep_the_plain_tables():
    inp = _Inputs(GRAPHS["trailing_tails"](), _dev())
    plan = inp.plan(True)
    meta = {"type_count": plan.type_count, "sorted": True, "pairs": plan.pairs}
    free = P.build_plan(inp.nt, inp.ei, inp.et, inp.tm, T, R, host_meta=meta)
    assert free.dst_extent == free.type_count[:T]
    assert P.layer_tables(free, D, D, dst=True) is P.layer_tables(free, D, D)


def test_training_gradients_do_not_depend_on_the_extents():
    inp = _Inputs(GRAPHS["trailing_tails"](), _dev())
    m = _module(True, True, dropout=0.0).train()
    plan = inp.plan(True)

    def run():
        m.zero_grad(set_to_none=True)
        x = inp.x.clone().requires_grad_(True)
        out = m(x, inp.nt, inp.ei, inp.et, inp.tm)
        (out * torch.linspace(-1, 1, D, device=out.device)).sum().backward()
        return (out.detach(), x.grad) + tuple(p.grad for p in m.parameters() if p.grad is not None)
    # the default backward adds gradients with float atomics, so only the deterministic one repeats bit for bit
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _assert_equal(*_both(plan, run), what="training output / gradient")
    finally:
        torch.use_deterministic_algorithms(prev)


def test_sharded_active_prefix_ignores_the_extents():
    inp = _Inputs(GRAPHS["trailing_tails"](), _dev())
    m = _module(True, False)
    plan = inp.plan(False)
    active = [c // 2 for c in plan.type_count[:T]]

    def run():
        with torch.no_grad():
            out, _, _ = m._forward_impl(inp.x, inp.nt, inp.ei, inp.et, None, want_att=False, save=False,
                                        active_per_type=active)
        return out
    assert P.layer_tables(plan, D, D, active, dst=True).type_dst_dev is None
    _assert_equal(*_both(plan, run), what="active-prefix output")


def test_trimmed_forward_ignores_the_extents():
    inp = _Inputs(GRAPHS["no_in_edges_first"](), _dev())
    torch.manual_seed(2)
    gnn = GNN(D, D, T, R, H, 2, dropout=0.2, use_RTE=True).to(_dev()).eval()
    plan = inp.plan(True)
    out_nodes = torch.arange(0, inp.g.num_nodes, 7, device=_dev())

    def run():
        with torch.no_grad():
            return gnn(inp.x, inp.nt, inp.tm, inp.ei, inp.et, out_nodes=out_nodes)
    _assert_equal(*_both(plan, run), what="trimmed output")
