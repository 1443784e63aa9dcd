"""Sharded training (ShardedGraph.forward_train, the path bench.py's c4 line trains through at --gpus N > 1) against
float64 autograd of the whole graph, with every rank of a W-way split emulated on one GPU in one process.

Emulation.  Every rank's ShardedGraph is built with (rank, W) on cuda:0 and gets its own deepcopy of the layers.  The real
forward_train runs for every rank, with sharded._HaloExchange replaced by _Emulation: it asserts that the rank's x_own is
bitwise X[owned_global] of the layer's global input X and returns X[local_global]; its backward index_copy's the local
gradient into zeros of X's shape (the local rows are unique), and autograd sums the ranks' contributions to X, which is
what the reverse all-to-all and the index_add of _HaloExchange.backward do.  The next layer's X is every rank's owned
output index_copy'd into one [N, d] tensor in rank order (the owned sets partition the nodes).  The per-rank parameter
gradients are summed in rank order in place of allreduce_grads.  The float64 reference is oracle.hgt_forward_ref_port on
the whole graph, chained layer by layer, and every case compares each rank's owned output rows, d X and every summed
parameter gradient (test_gpu_grad_parity._compare).  Free device memory is filled with NaN before every step, so a row a
kernel reads without anything having written it shows up as NaN instead of a stale value that may cancel.

Which projection tables a rank gets (plan.layer_tables): with kv_runs (ShardedGraph.build, num_relations <= 16) the
"compacted" tables, one Q group per type and one K'/V' group per row run of every <type, relation> pair, when there are at
most 64 such groups; their K'/V' groups overlap in rows, so the projection backward splits them into disjoint sub-tables,
the first writing dA and the later ones adding into it.  Otherwise the plain tables of the active prefixes.
_expected_tables restates that choice on the host; test_case_list_reaches_every_table_branch (no GPU needed) checks that
the cases below reach every branch, and every GPU run asserts the branch each rank took.

  c4        bench.py's c4 layer (d 256, H 8, use_norm, no RTE) as a 3-layer stack on make_mag_shaped(0.002,
            dst_zipf=1.2) plus two hubs above plan.TILE_SPLIT_EDGES fed from the far end of the paper ids (mostly halo
            rows), W = 2, 4, 8, linear_impl 0 and 1: every rank compacted, 8-12 groups, 3 backward sub-tables
  t4r4_rte  one d 512 / H 8 layer with RTE on test_gpu_grad_parity._graph(4, 4), W = 8: compacted, 32-64 groups (two
            ranks at exactly 64), 3-5 sub-tables
  t4r8      R = 8, W = 4: more than 64 groups, so the plain tables
  r17       R = 17, W = 4: kv_runs is None
  edges     node types >= T and relations >= R mixed in, a type with no nodes, a type with fewer nodes than W (ranks
            with active[t] == 0 that hold halo rows of it), a rank whose owned nodes have no in-edges (no local edges
            at all), W = 8: compacted, 3-41 groups, 1-5 sub-tables

Bounds (relative Frobenius: out and d X, parameters) are those of the matching single-GPU cases of
test_gpu_grad_parity.  Worst errors observed on an H100 SXM (80 GB HBM3, 700 W power limit) over every run of a case,
deterministic ones included, as (out / d X, parameters): c4 impl 0 1.8e-6, 1.4e-5 (relation_pri); c4 impl 1 1.9e-7,
1.7e-6 (skip); t4r4_rte 2.1e-6, 1.1e-5; t4r8 2.5e-6, 1.1e-5; r17 2.1e-6, 1.0e-5; edges 1.2e-6, 9.6e-6.  The c4 stack at
W = 4 under bf16 autocast: out max-abs 9.6e-3, relative Frobenius 4.2e-4 (out), 2.6e-4 (d X), 3.4e-3 (worst parameter,
skip); at "medium": 1.5e-2, 7.8e-4, 9.2e-4, 5.1e-3.

What each deliberate fault is caught by:
  later projection-backward sub-tables overwrite dA     test_sharded_training_matches_float64 (c4 with linear_impl 0,
  instead of adding into it                             t4r4_rte, edges), test_deterministic_steps_are_bitwise_equal_
                                                        and_lean_is_keep, test_c4_stack_under_reduced_precision_matches_
                                                        float64; not the runs with one sub-table (linear_impl 1, whose
                                                        SIMT dX adds overlapping groups itself; t4r8; r17)
  a kv_runs run end one row short in ShardedGraph.build every compacted run of the three GPU tests
  type_active dropped from the update backward          every c4, t4r4_rte and edges run of the three GPU tests: the
                                                        never-written a_linear rows of the halo sources (NaN-filled)
                                                        turn their d X into NaN
"""
import contextlib
import copy

import pytest
import torch

from pyhgt_b200 import plan as P, sharded, synth
from tests.test_gpu_grad_parity import (FRO_BOUND, _compare, _compare_all, _deterministic, _f64_params, _graph,
                                        _layer, _oracle_layer)


# ---------------------------------------------------------------------------------------------------------------------
# graphs

def _mag_graph():
    """make_mag_shaped(0.002, dst_zipf=1.2): 3.9 k nodes, 42 k edges, Zipf hubs; plus a paper hub (1500 'cites') and a
    field hub (2600 'has_topic') near the start of their types, fed from the upper three quarters of the paper ids, so
    that most of their sources are halo rows on the hub's rank at every W."""
    g = synth.make_mag_shaped(0.002, dst_zipf=1.2)
    gen = torch.Generator().manual_seed(7)
    papers = (g.node_type == 0).nonzero(as_tuple=True)[0]
    fields = (g.node_type == 3).nonzero(as_tuple=True)[0]
    far = papers[papers.numel() // 4:]
    src, dst, rel = [g.edge_index[0]], [g.edge_index[1]], [g.edge_type]
    for hub, cnt, r in ((papers[5], 1500, 1), (fields[3], 2600, 2)):
        assert cnt > P.TILE_SPLIT_EDGES
        src.append(far[torch.randint(0, far.numel(), (cnt,), generator=gen)])
        dst.append(torch.full((cnt,), int(hub), dtype=torch.int64))
        rel.append(torch.full((cnt,), r, dtype=torch.int64))
    g.edge_index = torch.stack([torch.cat(src), torch.cat(dst)])
    g.edge_type = torch.cat(rel)
    g.edge_time = torch.randint(0, 240, (g.edge_type.numel(),), generator=gen)
    g.hubs = (int(papers[5]), int(fields[3]))
    return g


def _edge_graph():
    """T = 4, R = 4, unsorted node order: 3000 nodes of type 0, none of type 1, 5 of type 2 and 900 of type 3, plus 150
    of the unknown type T + 2; every 7th edge has the unknown relation R + 5.  Only the lowest 40% of the ids of every
    type (the unknown one included) are destinations, so the last rank of an 8-way split owns isolated nodes only.  The
    5 nodes of type 2 feed 60 edges each: ranks without a node of type 2 hold halo rows of it.  One type-0 hub above
    TILE_SPLIT_EDGES."""
    T, R = 4, 4
    gen = torch.Generator().manual_seed(91)
    counts = ((0, 3000), (2, 5), (3, 900), (T + 2, 150))
    nt = torch.cat([torch.full((c,), t, dtype=torch.int64) for t, c in counts])
    nt = nt[torch.randperm(nt.numel(), generator=gen)]
    n = nt.numel()
    pools = [(nt == t).nonzero(as_tuple=True)[0][:max(1, int(0.4 * c))] for t, c in counts]
    pool = torch.cat(pools)
    few = (nt == 2).nonzero(as_tuple=True)[0]
    n_rand, n_hub = 5000, 1500
    assert n_hub > P.TILE_SPLIT_EDGES
    src = torch.cat([torch.randint(0, n, (n_rand,), generator=gen), few.repeat_interleave(60),
                     torch.randint(0, n, (n_hub,), generator=gen)])
    dst = torch.cat([pool[torch.randint(0, pool.numel(), (n_rand + 60 * few.numel(),), generator=gen)],
                     torch.full((n_hub,), int(pools[0][0]), dtype=torch.int64)])
    rel = torch.randint(0, R, (src.numel(),), generator=gen)
    rel[::7] = R + 5
    tm = torch.randint(0, 240, (src.numel(),), generator=gen)
    return synth.HeteroGraph(nt, torch.stack([src, dst]), rel, tm, T, R, "edges")


# name: (graph, d, n_heads, use_RTE, layers, (out and d X bound, parameter bound))
CASES = {
    "c4": (_mag_graph, 256, 8, False, 3, (5e-5, 1e-4)),        # test_c4_three_layer_stack_matches_float64
    "t4r4_rte": (lambda: _graph(4, 4, 0, False), 512, 8, True, 1, FRO_BOUND["mag_d512_h8_rte"]),
    "t4r8": (lambda: _graph(4, 8, 5, False), 128, 8, False, 1, FRO_BOUND["c5_d128_h8"]),
    "r17": (lambda: _graph(4, 17, 6, False), 128, 8, True, 1, FRO_BOUND["c5_d128_h8"]),
    "edges": (_edge_graph, 256, 8, True, 1, (3e-5, 3e-4)),     # test_unmatched_edges_backward_matches_float64
}
# (case, W, linear_impl): linear_impl 1 (SIMT GEMMs, whose dX adds overlapping groups itself) for c4 only
RUNS = [("c4", w, impl) for w in (2, 4, 8) for impl in (0, 1)] + [("t4r4_rte", 8, 0), ("t4r8", 4, 0), ("r17", 4, 0),
                                                                   ("edges", 8, 0)]


def _build_shards(g, rte, world, dev):
    return [sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time if rte else None,
                                       g.num_types, g.num_relations, r, world, dev) for r in range(world)]


# ---------------------------------------------------------------------------------------------------------------------
# the projection tables a rank gets

def _expected_tables(sh):
    """plan.layer_tables' choice for a shard's local graph, restated on the host: (branch, groups, backward sub-tables),
    branch "kv_runs None", "fallback" (kv_runs given, plain tables) or "compacted"."""
    T, R = sh.num_types, sh.num_relations
    nt, et = sh.node_type.cpu(), sh.edge_type.cpu()
    src, dst = sh.edge_index.cpu()
    count = [int((nt == t).sum()) for t in range(T)]
    row0 = [sum(count[:t]) for t in range(T)]

    def known(v, n):
        return (v >= 0) & (v < n)

    sel = known(nt[src], T) & known(nt[dst], T) & known(et, R)
    pairs = sorted(set(zip(nt[src][sel].tolist(), et[sel].tolist())))      # plan.pairs
    act = [min(int(a), c) for a, c in zip(sh.active_per_type, count)]
    q = [(row0[t], act[t]) for t in range(T) if count[t] and act[t]]
    groups = q + [(row0[t] + act[t], count[t] - act[t]) for t in range(T)
                  if count[t] > act[t] and any(s == t for s, _ in pairs)]
    branch = "kv_runs None" if sh.kv_runs is None else "fallback"
    if sh.kv_runs is not None:
        runs = dict(sh.kv_runs)
        g2 = q + [(row0[s] + r0, min(r1, count[s]) - r0) for s, r in pairs for r0, r1 in runs.get((s, r), ())
                  if min(r1, count[s]) > r0]
        if len(g2) <= 64 and all(p in runs for p in pairs):
            groups, branch = g2, "compacted"
    subsets = []                                   # greedy colouring into sub-tables of row-disjoint groups
    for a0, m in sorted(groups, key=lambda g_: (g_[0], g_[0] + g_[1])):
        for sub in subsets:
            if all(a0 >= b0 + n_ or b0 >= a0 + m for b0, n_ in sub):
                sub.append((a0, m))
                break
        else:
            subsets.append([(a0, m)])
    return branch, len(groups), max(len(subsets), 1)


def _branch_labels(branch, n_groups, n_sub):
    labels = {branch}
    if branch == "compacted" and n_groups == 64:
        labels.add("compacted, 64 groups")
    if branch == "compacted" and n_sub >= 2:
        labels.add("compacted, >= 2 sub-tables")
    return labels


def test_case_list_reaches_every_table_branch():
    """The runs reach every branch of plan.layer_tables; the c4 runs (bench.py's path) are compacted with several
    backward sub-tables on every rank."""
    cpu = torch.device("cpu")
    seen, per_case = set(), {}
    for name, world in sorted({(n, w) for n, w, _ in RUNS}):
        graph, _, _, rte, _, _ = CASES[name]
        for sh in _build_shards(graph(), rte, world, cpu):
            got = _expected_tables(sh)
            seen |= _branch_labels(*got)
            per_case.setdefault(name, []).append(got)
    assert seen == {"kv_runs None", "fallback", "compacted", "compacted, 64 groups", "compacted, >= 2 sub-tables"}, seen
    assert all(b == "compacted" and n_sub >= 2 for b, _, n_sub in per_case["c4"]), per_case["c4"]
    assert sum(b == "compacted" and n == 64 for b, n, _ in per_case["t4r4_rte"]) >= 2, per_case["t4r4_rte"]
    assert all(b == "fallback" for b, _, _ in per_case["t4r8"])
    assert all(b == "kv_runs None" for b, _, _ in per_case["r17"])


def test_hubs_and_edge_cases_are_present():
    """The c4 hubs are split destinations whose sources are mostly halo rows at every W; the edge graph has the shapes
    its docstring lists."""
    cpu = torch.device("cpu")
    g = _mag_graph()
    deg = torch.bincount(g.edge_index[1], minlength=g.num_nodes)
    for world in (2, 4, 8):
        for sh in _build_shards(g, False, world, cpu):
            halo = torch.ones(sh.n_owned + sh.n_halo, dtype=torch.bool)
            halo[sh.own_rows] = False
            for hub in g.hubs:
                if hub in sh.owned_global:
                    assert int(deg[hub]) > P.TILE_SPLIT_EDGES
                    share = halo[sh.edge_index[0][sh.local_global[sh.edge_index[1]] == hub]].float().mean()
                    assert share > 0.5, (world, sh.rank, hub, share)
    g = _edge_graph()
    T = g.num_types
    assert (g.node_type >= T).sum() == 150 and (g.edge_type >= g.num_relations).sum() > 900
    assert (g.node_type == 1).sum() == 0 and 0 < (g.node_type == 2).sum() < 8
    assert int(torch.bincount(g.edge_index[1]).max()) > P.TILE_SPLIT_EDGES
    shs = _build_shards(g, True, 8, cpu)
    assert any(sh.active_per_type[2] == 0 and (sh.node_type == 2).any() for sh in shs)
    assert any(sh.n_local_edges == 0 and sh.active_per_type[0] > 0 for sh in shs)


# ---------------------------------------------------------------------------------------------------------------------
# the emulated split

class _Gather(torch.autograd.Function):
    """X[rows]; backward: the gradient index_copy'd into zeros of X's shape (rows are unique: no atomics)."""

    @staticmethod
    def forward(ctx, x, rows):
        ctx.save_for_backward(rows)
        ctx.n = x.shape[0]
        return x.index_select(0, rows)

    @staticmethod
    def backward(ctx, d_rows):
        rows, = ctx.saved_tensors
        dx = torch.zeros((ctx.n, d_rows.shape[1]), dtype=d_rows.dtype, device=d_rows.device)
        return dx.index_copy_(0, rows, d_rows), None


class _Emulation:
    """Every rank of a W-way split in this process.  Installed as sharded._HaloExchange: `apply(x_own, shard)` is the halo
    exchange of one rank for the layer whose global input is `self.X`."""

    def __init__(self, g, rte, world, dev):
        self.shards = _build_shards(g, rte, world, dev)
        self.own = [sh.owned_global.to(dev) for sh in self.shards]
        self.local = {id(sh): (o, sh.local_global.to(dev)) for sh, o in zip(self.shards, self.own)}
        self.own_cat = torch.cat(self.own)
        assert torch.equal(torch.sort(self.own_cat)[0].cpu(), torch.arange(g.num_nodes))   # a partition
        self.X = None

    def apply(self, x_own, sh):
        own, local = self.local[id(sh)]
        bits = torch.int32
        assert torch.equal(x_own.detach().view(bits), self.X.detach().index_select(0, own).view(bits)), \
            "rank %d: x_own is not bitwise X[owned_global]" % sh.rank
        return _Gather.apply(self.X, local)

    def assemble(self, outs):
        """[N, d] with every rank's owned output rows at their global rows."""
        cat = torch.cat(outs)
        return torch.zeros((self.own_cat.numel(), cat.shape[1]), dtype=cat.dtype,
                           device=cat.device).index_copy(0, self.own_cat, cat)


def _poison_free_memory(dev):
    """Fill the caching allocator's free memory with NaN (1 GB of large blocks, 64 MB of small ones)."""
    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    big = [torch.full((1 << 26,), float("nan"), device=dev) for _ in range(4)]
    small = [torch.full((1 << 18,), float("nan"), device=dev) for _ in range(64)]
    torch.cuda.synchronize(dev)
    del big, small


_CACHE = {}


def _reference(name):
    """Graph, layers (CPU), input, loss weight and the float64 result of one case, computed once."""
    if name not in _CACHE:
        graph, d, H, rte, L, _ = CASES[name]
        g = graph()
        seed = sum(map(ord, name)) % 1000
        layers = torch.nn.ModuleList([_layer(d, H, g.num_types, g.num_relations, rte, seed + 2 * i) for i in range(L)])
        x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(seed + 100))
        w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(seed + 101))
        params = [_f64_params(m) for m in layers]
        xr = x.double().requires_grad_(True)
        h = xr
        for p, m in zip(params, layers):
            h = _oracle_layer(p, h, g, m)
        (h * w.double()).sum().backward()
        ref = (h.detach(), xr.grad, {"%d.%s" % (i, k): v.grad for i, p in enumerate(params) for k, v in p.items()})
        _CACHE[name] = (g, layers, x, w, ref)
    return _CACHE[name]


def _setup(name, world, impl, monkeypatch):
    """(emulation, per-rank layer copies, x, w, float64 result), with the emulation installed as the halo exchange."""
    import pyhgt_b200
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, layers, x, w, ref = _reference(name)
    emu = _Emulation(g, CASES[name][3], world, dev)
    monkeypatch.setattr(sharded, "_HaloExchange", emu)
    copies = []
    for _ in range(world):
        c = copy.deepcopy(layers).to(dev).train()
        for m in c:
            m.linear_impl = impl
        copies.append(c)
    return emu, copies, x.to(dev), w.to(dev), ref


def _step(emu, copies, x, w, lean=False):
    """One emulated training step, loss = sum(out * w): (every rank's owned output rows, d X, every rank's parameter
    gradients)."""
    for c in copies:
        c.zero_grad(set_to_none=True)
        for m in c:
            m.recompute_tables = lean
    _poison_free_memory(x.device)
    X = x.clone().requires_grad_(True)
    h = X
    outs = [X.detach().index_select(0, o) for o in emu.own]
    for layer in range(len(copies[0])):
        emu.X = h
        outs = [sh.forward_train(c[layer], o) for sh, c, o in zip(emu.shards, copies, outs)]
        h = emu.assemble(outs)
    (h * w).sum().backward()
    torch.cuda.synchronize()
    grads = [{k: None if p.grad is None else p.grad.clone() for k, p in c.named_parameters()} for c in copies]
    return [o.detach().clone() for o in outs], X.grad, grads


def _summed(grads):
    """Every parameter's gradient summed over the ranks in rank order (allreduce_grads)."""
    total = {}
    for k in grads[0]:
        parts = [g[k] for g in grads if g[k] is not None]
        total[k] = None
        for p in parts:
            total[k] = p.clone() if total[k] is None else total[k] + p
    return total


def _check_tables(emu, copies):
    """Every rank took the projection tables _expected_tables predicts."""
    m = copies[0][0]
    for sh in emu.shards:
        pl = P.get_plan(sh.node_type, sh.edge_index, sh.edge_type, sh.edge_time if m.use_RTE else None,
                        m.num_types, m.num_relations)
        lt = P.layer_tables(pl, m.in_dim, m.out_dim, sh.active_per_type, sh.kv_runs)
        branch, n_groups, n_sub = _expected_tables(sh)
        got = (lt.proj_groups[2], len(lt.proj_groups.bwd_tables))
        assert got == (n_groups, n_sub), "rank %d: %s tables expected %s, got %s" % (sh.rank, branch,
                                                                                      (n_groups, n_sub), got)


def _compare_ranks(tag, emu, native, ref, bounds):
    """Each rank's owned output rows, d X and the summed parameter gradients against float64."""
    outs, dx, grads = native
    for sh, o, own in zip(emu.shards, outs, emu.own):
        if sh.n_owned:
            _compare(o, ref[0][own.cpu()], "%s rank %d out" % (tag, sh.rank), bounds[0])
    _compare_all(tag, (emu.assemble(outs), dx, _summed(grads)), ref, bounds)


@pytest.mark.gpu
@pytest.mark.parametrize("name,world,impl", RUNS)
def test_sharded_training_matches_float64(name, world, impl, monkeypatch):
    emu, copies, x, w, ref = _setup(name, world, impl, monkeypatch)
    native = _step(emu, copies, x, w)
    _check_tables(emu, copies)
    _compare_ranks("%s W=%d impl %d" % (name, world, impl), emu, native, ref, CASES[name][5])


def _assert_bitwise(a, b, tag):
    (oa, dxa, ga), (ob, dxb, gb) = a, b
    for r, (x, y) in enumerate(zip(oa, ob)):
        assert torch.equal(x, y), "%s: rank %d output" % (tag, r)
    assert torch.equal(dxa, dxb), "%s: d X" % tag
    for r, (x, y) in enumerate(zip(ga, gb)):
        bad = [k for k in sorted(x) if not ((x[k] is None and y[k] is None) or torch.equal(x[k], y[k]))]
        assert not bad, "%s: rank %d gradients differ: %s" % (tag, r, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("c4", 4), ("t4r4_rte", 8)])
def test_deterministic_steps_are_bitwise_equal_and_lean_is_keep(name, world, monkeypatch):
    """Under torch.use_deterministic_algorithms two emulated steps are bitwise equal on every rank, the lean step
    (recompute_tables) is bitwise the keep step on every rank, and both match float64."""
    emu, copies, x, w, ref = _setup(name, world, 0, monkeypatch)
    with _deterministic(True):
        keep = _step(emu, copies, x, w)
        again = _step(emu, copies, x, w)
        lean = _step(emu, copies, x, w, lean=True)
    _check_tables(emu, copies)
    _assert_bitwise(keep, again, "%s W=%d two keep steps" % (name, world))
    _assert_bitwise(keep, lean, "%s W=%d lean vs keep" % (name, world))
    _compare_ranks("%s W=%d deterministic" % (name, world), emu, keep, ref, CASES[name][5])


def _rel(got, ref):
    got, ref = got.detach().cpu().double(), ref.detach().double()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16_autocast", "medium"])
def test_c4_stack_under_reduced_precision_matches_float64(mode, monkeypatch):
    """The c4 stack at W = 4 under bf16 autocast (bf16 K'/V' tables) and at set_float32_matmul_precision("medium") (one
    bf16 product per GEMM), against float64 with the bounds of test_gpu_bf16_tables / test_gpu_matmul_precision:
    outputs max-abs 5e-2 and relative Frobenius 1e-2, gradients relative Frobenius 5e-2 (bf16) / 2e-2 (medium)."""
    from tests.test_gpu_bf16_tables import OUT_MAX_ABS, OUT_REL_FRO
    from tests.test_gpu_matmul_precision import GRAD_REL_FRO
    grad_bound = 5e-2 if mode == "bf16_autocast" else GRAD_REL_FRO
    emu, copies, x, w, ref = _setup("c4", 4, 0, monkeypatch)
    prec = torch.get_float32_matmul_precision()
    ctx = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "bf16_autocast" else contextlib.nullcontext()
    try:
        if mode == "medium":
            torch.set_float32_matmul_precision("medium")
        with ctx:
            outs, dx, grads = _step(emu, copies, x, w)
    finally:
        torch.set_float32_matmul_precision(prec)
    _check_tables(emu, copies)
    out = emu.assemble(outs).cpu().double()
    assert torch.isfinite(out).all()
    err, fro = float((out - ref[0]).abs().max()), _rel(out, ref[0])
    assert err <= OUT_MAX_ABS and fro <= OUT_REL_FRO, "%s: out max-abs %.3g, rel-Frobenius %.3g" % (mode, err, fro)
    errs = {}
    for k, g in [("d X", dx)] + sorted(_summed(grads).items()):
        r = ref[1] if k == "d X" else ref[2][k]
        if r is None or not r.abs().max():
            assert g is None or not g.abs().max(), "%s: %s: float64 gradient is zero, native is not" % (mode, k)
            continue
        assert g is not None and torch.isfinite(g).all(), "%s: %s" % (mode, k)
        errs[k] = _rel(g, r)
        assert errs[k] <= grad_bound, "%s: %s relative Frobenius %.3g" % (mode, k, errs[k])
    worst = max((k for k in errs if k != "d X"), key=errs.get)
    print("\n%s: out max-abs %.2e, rel fro out %.2e, d X %.2e, worst parameter %.2e (%s)"
          % (mode, err, fro, errs["d X"], errs[worst], worst))
