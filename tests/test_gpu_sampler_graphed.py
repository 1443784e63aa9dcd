"""sampler.GraphedSampler: fixed-shape sampling with no read-back, bitwise the unbounded chain
sample_subgraphs_cuda -> merge_batches (members > 1) -> the graphed classes' scatter into the signature's layout."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

pytestmark = pytest.mark.gpu

TIME_RANGE = {y: True for y in range(1990, 2016)}           # OAG-style training years
PAPER_FIELD = {("paper", "field", "PF_in_L2"): (128, 0), ("field", "paper", "rev_PF_in_L2"): (0, 128)}


@pytest.fixture(scope="module")
def graphs():
    from gpu_sampler_bench import make_graph
    from pyhgt_b200 import sampler
    dev = torch.device("cuda:0")
    g, n, year, _ = make_graph(0.05, seed=3)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(5)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), 24).astype(np.float32)) for t in n}
    out = {"fp32": sampler.DeviceGraph(fg, dev, tables),
           "bf16": sampler.DeviceGraph(fg, dev, tables, feature_dtype=torch.bfloat16)}
    return out, n, year


def _seeds(n, year, seed, count=128):
    rng = np.random.RandomState(seed)
    ids = rng.choice(n["paper"], count, replace=False)
    return {"paper": np.stack([ids, year[ids]], 1)}


def _keys(seed, B):
    g = torch.Generator()
    g.manual_seed(seed)
    return [int(torch.randint(0, 2 ** 63 - 1, (1,), generator=g)) for _ in range(B)]


def _unbounded(dg, sig, depth, W, inp, B, seed, time_range, mask, fdt):
    """sample_subgraphs_cuda -> merge_batches -> _Graphed._scatter, plus node_id / node_time in signature rows."""
    from pyhgt_b200 import graphed, sampler
    g = torch.Generator()
    g.manual_seed(seed)
    out = sampler.sample_subgraphs_cuda(dg, time_range, depth, W, [inp] * B, g, edge_mask=mask, feature_dtype=fdt)
    T, R = len(dg.types), len(dg.edge_dict)
    if B > 1:
        nf, nt, etime, ei, et, member_rows = sampler.merge_batches(out, T, R)
        batch = (nf, nt, etime, ei, et)
    else:
        batch = out[0][:5]
        member_rows = [torch.arange(out[0][1].shape[0], device=dg.device)]
    gr = graphed._Graphed(sig, dg.device)
    gr.stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(gr.stream):
        rows = gr._scatter(batch, *graphed.device_batch_sizes(sig, *batch))
    torch.cuda.synchronize()
    node_id = torch.full((sig.n_nodes,), -1, dtype=torch.int64, device=dg.device)
    node_time = torch.zeros(sig.n_nodes, dtype=torch.int64, device=dg.device)
    for b, mb in enumerate(out):
        indxs, times = mb[7], mb[8]
        present = [t for t in dg.types if t in indxs]
        srow = rows[member_rows[b]]
        if present:
            node_id[srow] = torch.cat([indxs[t] for t in present])
            node_time[srow] = torch.cat([times[t] for t in present])
    return {"x": gr.x, "ei": gr.ei, "et": gr.et, "tm": gr.tm, "node_id": node_id, "node_time": node_time}


def _assert_same(gs, ref):
    for k, v in ref.items():
        got = getattr(gs, k)
        assert got.shape == v.shape and got.dtype == v.dtype, k
        if got.dtype in (torch.float32, torch.bfloat16):
            assert torch.equal(got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                               v.view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32)), k
        else:
            assert torch.equal(got, v), k


def _signature(dg, depth, W, probes, B, time_range, mask, fdt):
    from pyhgt_b200 import sampler
    return sampler.graph_signature_for(dg, depth, W, probes, 0.5, members=B, time_range=time_range, edge_mask=mask,
                                       feature_dtype=fdt)


@pytest.mark.parametrize("shape", [(3, 64), (6, 520)])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("layout", ["dense", "hashed"])
@pytest.mark.parametrize("time_on", [True, False])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_fill_equals_the_unbounded_chain_bitwise(graphs, shape, B, layout, time_on, masked, dtype, monkeypatch):
    from pyhgt_b200 import sampler
    dgs, n, year = graphs
    dg = dgs[dtype]
    fdt = torch.bfloat16 if dtype == "bf16" else None
    depth, W = shape
    tr = TIME_RANGE if time_on else None
    mask = PAPER_FIELD if masked else None
    probes = [_seeds(n, year, s) for s in range(3)]
    sig = _signature(dg, depth, W, probes, B, tr, mask, fdt)
    gs = sampler.GraphedSampler(dg, sig, depth, W, {"paper": 128}, members=B, time_range=tr, edge_mask=mask,
                                feature_dtype=fdt)
    monkeypatch.setattr(sampler, "_FORCE_LAYOUT", layout)
    for s in (11, 12):
        inp = _seeds(n, year, s)
        gs.fill(inp, torch.tensor(_keys(s, B), dtype=torch.int64, device=dg.device))
        gs.check()
        _assert_same(gs, _unbounded(dg, sig, depth, W, inp, B, s, tr, mask, fdt))


def test_fewer_seeds_than_declared_and_two_seed_types(graphs):
    from pyhgt_b200 import sampler
    dgs, n, year = graphs
    dg = dgs["fp32"]
    inp = _seeds(n, year, 4, count=50)
    inp["author"] = np.stack([np.arange(7) * 13, np.full(7, 2000)], 1)
    sig = _signature(dg, 4, 64, [inp], 2, TIME_RANGE, None, None)
    gs = sampler.GraphedSampler(dg, sig, 4, 64, {"author": 10, "paper": 128}, members=2, time_range=TIME_RANGE)
    gs.fill(inp, torch.tensor(_keys(9, 2), dtype=torch.int64, device=dg.device))
    gs.check()
    _assert_same(gs, _unbounded(dg, sig, 4, 64, inp, 2, 9, TIME_RANGE, None, None))


def test_captured_fill_resamples_at_every_replay(graphs):
    from pyhgt_b200 import sampler
    dgs, n, year = graphs
    dg = dgs["fp32"]
    B = 3
    sig = _signature(dg, 6, 520, [_seeds(n, year, s) for s in range(3)], B, TIME_RANGE, None, None)
    gs = sampler.GraphedSampler(dg, sig, 6, 520, {"paper": 128}, members=B, time_range=TIME_RANGE)
    gs.fill(_seeds(n, year, 0), torch.tensor(_keys(0, B), dtype=torch.int64, device=dg.device))   # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gs.run()
    for s in (21, 22):
        inp = _seeds(n, year, s)
        gs.stage(inp)
        gs.copy_in(torch.tensor(_keys(s, B), dtype=torch.int64, device=dg.device))
        graph.replay()
        graph.replay()                                     # a replay without a new copy_in samples the same batch
        torch.cuda.synchronize()
        gs.check()
        _assert_same(gs, _unbounded(dg, sig, 6, 520, inp, B, s, TIME_RANGE, None, None))


def test_fill_does_not_synchronise(graphs):
    from pyhgt_b200 import sampler
    dgs, n, year = graphs
    dg = dgs["bf16"]
    sig = _signature(dg, 3, 64, [_seeds(n, year, 1)], 2, None, None, torch.bfloat16)
    gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128}, members=2, feature_dtype=torch.bfloat16)
    gs.fill(_seeds(n, year, 1))                            # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        gs.fill(_seeds(n, year, 2))
        gs.fill(_seeds(n, year, 3))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    gs.check()
    assert int((gs.node_id >= 0).sum()) > 0


def _exact_signature(dg, depth, W, inp, key_seed):
    from pyhgt_b200 import graphed, plan, sampler
    g = torch.Generator()
    g.manual_seed(key_seed)
    b = sampler.sample_subgraph_cuda(dg, None, depth, W, inp, g)
    T, R = len(dg.types), len(dg.edge_dict)
    p = plan.get_plan(b[1], b[3], b[4], b[2], T, R)
    return [int(c) for c in p.type_count[:T]], int(p.n_edges), sampler._mag_pairs(dg)


@pytest.mark.parametrize("short", ["edge", "node", "room"])
def test_a_bound_overflow_poisons_the_features_and_check_names_it(graphs, short):
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = graphs
    dg = dgs["fp32"]
    inp = _seeds(n, year, 7)
    counts, E, pairs = _exact_signature(dg, 3, 64, inp, 7)
    R = len(dg.edge_dict)
    exact = graphed.GraphSignature(counts, E, pairs, R, dg.feat_dim)
    gs = sampler.GraphedSampler(dg, exact, 3, 64, {"paper": 128})
    keys = torch.tensor(_keys(7, 1), dtype=torch.int64, device=dg.device)
    gs.fill(inp, keys)
    gs.check()                                             # the exact signature fits
    assert not torch.isnan(gs.x).any()
    room = dg.state_room
    if short == "edge":
        sig, match = graphed.GraphSignature(counts, E - 1, pairs, R, dg.feat_dim), "more edges"
    elif short == "node":
        t = dg.slot["author"]
        sig = graphed.GraphSignature([c - (i == t) for i, c in enumerate(counts)], E, pairs, R, dg.feat_dim)
        match = "node type 'author'"
    else:
        sig, match = exact, "hashed state region"
        dg.state_room = 0.05
    try:
        gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128})
    finally:
        dg.state_room = room
    gs.fill(inp, keys)
    assert torch.isnan(gs.x).all()
    assert int((gs.node_id >= 0).sum()) == 0              # nothing laid out
    with pytest.raises(ValueError, match=match):
        gs.check()


def _small_graph(adj):
    from tests.test_gpu_sampler import _small
    from pyhgt_b200 import sampler
    g = _small(adj)
    fg = sampler.FrozenGraph(g)
    tabs = {t: torch.ones(max(fg.n_ids.get(t, 1), 1), 4) for t in ("paper", "author")}
    return fg, sampler.DeviceGraph(fg, torch.device("cuda:0"), tabs)


def _loose_signature(dg):
    from pyhgt_b200 import graphed, sampler
    return graphed.GraphSignature([16] * len(dg.types), 64, sampler._mag_pairs(dg), len(dg.edge_dict), dg.feat_dim)


def test_range_errors_raise_what_the_unbounded_path_raises():
    """edge_time: seed papers at 2000 and a seed author at 2200 (test_gpu_sampler_mask's case); neighbour ids: an author
    id range declared below the authors the papers list."""
    from pyhgt_b200 import sampler
    _, dg = _small_graph({0: [10, 11], 1: [10]})
    inp = {"paper": np.array([[0, 2000], [1, 2000]]), "author": np.array([[10, 2200]])}
    with pytest.raises(IndexError, match="edge_time") as ref:
        sampler.sample_subgraph_cuda(dg, {2000: True}, 0, 4, inp)
    gs = sampler.GraphedSampler(dg, _loose_signature(dg), 0, 4, {"paper": 2, "author": 1}, time_range={2000: True})
    gs.fill(inp)
    with pytest.raises(IndexError) as got:
        gs.check()
    assert str(got.value) == str(ref.value)
    assert torch.isnan(gs.x).all()

    _, dg = _small_graph({0: [10, 11], 1: [10]})
    dg.n_ids = list(dg.n_ids)
    dg.n_ids[dg.slot["author"]] = 5
    inp = {"paper": np.array([[0, 2000], [1, 2000]])}
    with pytest.raises(IndexError, match="neighbour id") as ref:
        sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 4, inp)
    gs = sampler.GraphedSampler(dg, _loose_signature(dg), 1, 4, {"paper": 2}, time_range={2000: True})
    gs.fill(inp)
    with pytest.raises(IndexError) as got:
        gs.check()
    assert str(got.value) == str(ref.value)
    assert torch.isnan(gs.x).all()


@pytest.mark.parametrize("short", ["edge", "node"])
def test_an_overflow_writes_nothing_past_any_buffer(graphs, short):
    """Every output is a view at the head of a larger buffer whose tail holds a sentinel; an overflowing fill (and a
    fitting one) must leave every tail as it was."""
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = graphs
    for dtype in ("fp32", "bf16"):
        dg = dgs[dtype]
        fdt = torch.bfloat16 if dtype == "bf16" else None
        inp = _seeds(n, year, 8)
        counts, E, pairs = _exact_signature(dg, 3, 64, inp, 8)
        R = len(dg.edge_dict)
        if short == "edge":
            E -= 1
        else:
            counts[dg.slot["paper"]] -= 1
        sig = graphed.GraphSignature(counts, E, pairs, R, dg.feat_dim,
                                     feat_dtype=torch.bfloat16 if fdt else torch.float32)
        gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128}, feature_dtype=fdt)
        tails = {}
        for name in ("x", "nt", "ei", "et", "tm", "node_id", "node_time"):
            t = getattr(gs, name)
            big = torch.empty(t.numel() + 4096, dtype=t.dtype, device=t.device)
            big.view(torch.int16 if t.element_size() == 2 else (torch.int32 if t.element_size() == 4 else torch.int64)).fill_(0x5a5a)
            big[:t.numel()].copy_(t.reshape(-1))
            setattr(gs, name, big[:t.numel()].view(t.shape))
            tails[name] = (big, big[t.numel():].clone())
        for s in (8, 9):
            gs.fill(_seeds(n, year, s), torch.tensor(_keys(8, 1), dtype=torch.int64, device=dg.device))
        torch.cuda.synchronize()
        for name, (big, tail) in tails.items():
            assert torch.equal(big[-4096:].view(torch.int16 if big.element_size() == 2 else torch.uint8),
                               tail.view(torch.int16 if big.element_size() == 2 else torch.uint8)), name
        with pytest.raises(ValueError):
            gs.fill(inp, torch.tensor(_keys(8, 1), dtype=torch.int64, device=dg.device))
            gs.check()


# ---------------------------------------------------------------------------------------------------------------------
# the sampler captured with the training step and the forward

def _model(dg, seed=0):
    from pyhgt_b200.model import GNN
    torch.manual_seed(seed)
    gnn = GNN(dg.feat_dim, 32, len(dg.types), len(dg.edge_dict), 4, 2, 0.0, "hgt", True, True, True).cuda()
    head = torch.nn.Linear(32, 7).cuda()
    return gnn, head


def _label_loss(gnn, head, ids_of, label, paper):
    import torch.nn.functional as F

    def loss(x, nt, tm, ei, et, tg):
        ids = ids_of()
        y = torch.where((ids >= 0) & (nt == paper), label[ids.clamp(min=0)], torch.full_like(ids, -100))
        return F.nll_loss(F.log_softmax(head(gnn(x, nt, tm, ei, et)), -1), y, ignore_index=-100)
    return loss


def _opt(params):
    return torch.optim.AdamW(params, lr=torch.tensor(1e-3, device="cuda"), capturable=True)


def test_graphed_train_step_with_sampler_equals_the_unbounded_feed():
    """Three steps of GraphedTrainStep(sampler=gs) with explicit keys leave the parameters bitwise where three steps of
    GraphedTrainStep fed sample_subgraph_cuda's batches (same keys) leave them; deterministic, no dropout."""
    import copy
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = _graphs_once()
    dg = dgs["fp32"]
    paper = dg.slot["paper"]
    label = torch.randint(0, 7, (n["paper"],), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    sig = _signature(dg, 3, 64, [_seeds(n, year, s) for s in range(3)], 1, TIME_RANGE, None, None)
    gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128}, time_range=TIME_RANGE)
    gnn, head = _model(dg)
    gnn2, head2 = copy.deepcopy(gnn), copy.deepcopy(head)
    p1 = list(gnn.parameters()) + list(head.parameters())
    p2 = list(gnn2.parameters()) + list(head2.parameters())
    opt1, opt2 = _opt(p1), _opt(p2)
    ids_ref = torch.full((sig.n_nodes,), -1, dtype=torch.int64, device="cuda")
    step1 = graphed.GraphedTrainStep(_label_loss(gnn, head, lambda: gs.node_id, label, paper), sig, "cuda",
                                     optimizer=opt1, clip_norm=1.0, sampler=gs)
    step2 = graphed.GraphedTrainStep(_label_loss(gnn2, head2, lambda: ids_ref, label, paper), sig, "cuda",
                                     optimizer=opt2, clip_norm=1.0)
    torch.use_deterministic_algorithms(True)
    try:
        for s in (31, 32, 33):
            inp = _seeds(n, year, s)
            l1, = step1.step(inp, torch.tensor(_keys(s, 1), dtype=torch.int64, device="cuda"))
            ids_ref.copy_(_unbounded(dg, sig, 3, 64, inp, 1, s, TIME_RANGE, None, None)["node_id"])
            batch = sampler.sample_subgraph_cuda(dg, TIME_RANGE, 3, 64, inp, torch.Generator().manual_seed(s))
            l2, = step2(*batch[:5])
            torch.cuda.synchronize()
            assert torch.equal(l1, l2), s
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(p1, p2):
        assert torch.equal(a, b)


_GRAPHS = []


def _graphs_once():
    if not _GRAPHS:
        from gpu_sampler_bench import make_graph
        from pyhgt_b200 import sampler
        g, n, year, _ = make_graph(0.05, seed=3)
        fg = sampler.FrozenGraph(g)
        rng = np.random.RandomState(5)
        tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), 24).astype(np.float32)) for t in n}
        _GRAPHS.append(({"fp32": sampler.DeviceGraph(fg, torch.device("cuda:0"), tables)}, n, year))
    return _GRAPHS[0]


def test_graphed_training_from_the_sampler_reduces_the_loss_without_syncs():
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = _graphs_once()
    dg = dgs["fp32"]
    paper = dg.slot["paper"]
    label = torch.randint(0, 7, (n["paper"],), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    sig = _signature(dg, 3, 64, [_seeds(n, year, s) for s in range(3)], 1, None, None, None)
    gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128})
    gnn, head = _model(dg, 3)
    opt = torch.optim.AdamW(list(gnn.parameters()) + list(head.parameters()), lr=torch.tensor(1e-2, device="cuda"),
                            capturable=True)
    step = graphed.GraphedTrainStep(_label_loss(gnn, head, lambda: gs.node_id, label, paper), sig, "cuda",
                                    optimizer=opt, clip_norm=1.0, sampler=gs)
    seeds = [_seeds(n, year, s % 4) for s in range(40)]
    losses = []
    step.step(seeds[0])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for inp in seeds[1:]:
            losses.append(step.step(inp)[0].clone())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    gs.check()
    losses = [float(v) for v in losses]
    assert np.mean(losses[-5:]) < 0.9 * np.mean(losses[:5]), losses
    with pytest.raises(ValueError, match="step"):
        step(gs.x, gs.nt, gs.tm, gs.ei, gs.et)


def test_graphed_forward_with_eight_members_is_the_merged_forward():
    """GraphedForward(sampler=gs, members=8): one replay, bitwise the graphed forward of the merge_batches union of the
    unbounded sampler's 8 members, and close to the eager forward of that union."""
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = _graphs_once()
    dg = dgs["fp32"]
    B = 8
    sig = _signature(dg, 3, 64, [_seeds(n, year, 5)], B, TIME_RANGE, None, None)
    gs = sampler.GraphedSampler(dg, sig, 3, 64, {"paper": 128}, members=B, time_range=TIME_RANGE)
    gnn, _ = _model(dg, 4)
    gnn.eval()
    fn = lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et)
    fwd = graphed.GraphedForward(fn, sig, "cuda", sampler=gs)
    ref = graphed.GraphedForward(fn, sig, "cuda")
    for s in (41, 42):
        inp = _seeds(n, year, 5)
        out = fwd.step(inp, torch.tensor(_keys(s, B), dtype=torch.int64, device="cuda"))
        out_sync = out.clone()
        torch.cuda.synchronize()
        members = sampler.sample_subgraphs_cuda(dg, TIME_RANGE, 3, 64, [inp] * B, torch.Generator().manual_seed(s))
        merged = sampler.merge_batches(members, len(dg.types), len(dg.edge_dict))
        rows_out = ref(*merged[:5])                        # the union's rows, in union order
        with torch.no_grad():
            eager = fn(*merged[:5])
        exp = _unbounded(dg, sig, 3, 64, inp, B, s, TIME_RANGE, None, None)
        torch.cuda.synchronize()
        real = exp["node_id"] >= 0
        assert torch.equal(gs.node_id, exp["node_id"])
        assert int(real.sum()) == rows_out.shape[0]
        # signature rows of the union rows: type-contiguous in both, so the real rows in order are the union's rows
        assert torch.equal(out_sync[real], rows_out)
        assert torch.allclose(out_sync[real], eager, rtol=1e-4, atol=1e-4)
    torch.cuda.set_sync_debug_mode("error")
    try:
        fwd.step(_seeds(n, year, 6))
    finally:
        torch.cuda.set_sync_debug_mode(0)
