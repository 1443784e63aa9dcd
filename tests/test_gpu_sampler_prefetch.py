"""GraphedTrainStep.run / GraphedForward.run: batch k + 1 sampled on the sampler's prefetch stream while step k runs.
The results are bitwise those of the same batches through step(), with no host synchronisation, and a batch past the
signature is reported by its index in the run."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

pytestmark = pytest.mark.gpu

TIME_RANGE = {y: True for y in range(1990, 2016)}
PAPER_FIELD = {("paper", "field", "PF_in_L2"): (128, 0), ("field", "paper", "rev_PF_in_L2"): (0, 128)}
DEPTH, WIDTH = 3, 64
_GRAPHS = []


def _graphs():
    """The MAG-schema graph at scale 0.05 with fp32 and bf16 feature tables (built once per module)."""
    if not _GRAPHS:
        from gpu_sampler_bench import make_graph
        from pyhgt_b200 import sampler
        g, n, year, _ = make_graph(0.05, seed=3)
        fg = sampler.FrozenGraph(g)
        rng = np.random.RandomState(5)
        tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), 24).astype(np.float32)) for t in n}
        dev = torch.device("cuda:0")
        _GRAPHS.append(({"fp32": sampler.DeviceGraph(fg, dev, tables),
                         "bf16": sampler.DeviceGraph(fg, dev, tables, feature_dtype=torch.bfloat16)}, n, year))
    return _GRAPHS[0]


def _seeds(n, year, seed, count=128):
    rng = np.random.RandomState(seed)
    ids = rng.choice(n["paper"], count, replace=False)
    return {"paper": np.stack([ids, year[ids]], 1)}


def _keys(seeds, B):
    """[len(seeds), B] Philox keys on the device."""
    out = []
    for s in seeds:
        g = torch.Generator()
        g.manual_seed(s)
        out.append([int(torch.randint(0, 2 ** 63 - 1, (1,), generator=g)) for _ in range(B)])
    return torch.tensor(out, dtype=torch.int64, device="cuda")


def _model(dg, seed=0):
    from pyhgt_b200.model import GNN
    torch.manual_seed(seed)
    gnn = GNN(dg.feat_dim, 32, len(dg.types), len(dg.edge_dict), 4, 2, 0.0, "hgt", True, True, True).cuda()
    head = torch.nn.Linear(32, 7).cuda()
    return gnn, head


def _trainer(dg, sig, gnn, head, label, B, mask):
    """A GraphedTrainStep with its own GraphedSampler, labels read through the sampler's node_id."""
    import torch.nn.functional as F
    from pyhgt_b200 import graphed, sampler
    gs = sampler.GraphedSampler(dg, sig, DEPTH, WIDTH, {"paper": 128}, members=B, time_range=TIME_RANGE,
                                edge_mask=mask)
    paper = dg.slot["paper"]

    def loss(x, nt, tm, ei, et, tg):
        ids = gs.node_id
        y = torch.where((ids >= 0) & (nt == paper), label[ids.clamp(min=0)], torch.full_like(ids, -100))
        return F.nll_loss(F.log_softmax(head(gnn(x, nt, tm, ei, et)), -1), y, ignore_index=-100)
    params = list(gnn.parameters()) + list(head.parameters())
    opt = torch.optim.AdamW(params, lr=torch.tensor(1e-3, device="cuda"), capturable=True)
    return graphed.GraphedTrainStep(loss, sig, "cuda", optimizer=opt, clip_norm=1.0, sampler=gs), params


def _label(n):
    return torch.randint(0, 7, (n["paper"],), device="cuda", generator=torch.Generator("cuda").manual_seed(1))


def _two_trainers(dtype, B, mask, sig=None):
    from pyhgt_b200 import sampler
    dgs, n, year = _graphs()
    dg = dgs[dtype]
    if sig is None:
        sig = sampler.graph_signature_for(dg, DEPTH, WIDTH, [_seeds(n, year, s) for s in range(3)], 0.5, members=B,
                                          time_range=TIME_RANGE, edge_mask=mask)
    gnn, head = _model(dg)
    gnn2, head2 = copy.deepcopy(gnn), copy.deepcopy(head)
    label = _label(n)
    return (_trainer(dg, sig, gnn, head, label, B, mask), _trainer(dg, sig, gnn2, head2, label, B, mask), n, year)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(a, b):
    """Bitwise equal, NaN payloads included."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("masked", [False, True])
def test_run_trains_bitwise_like_step_calls(B, dtype, masked):
    """8 batches through run() leave losses and parameters bitwise where 8 step() calls leave them (same seeds and
    Philox keys, deterministic algorithms, dropout 0)."""
    (s1, p1), (s2, p2), n, year = _two_trainers(dtype, B, PAPER_FIELD if masked else None)
    seeds = list(range(60, 68))
    batches = [_seeds(n, year, s) for s in seeds]
    keys = _keys(seeds, B)
    torch.use_deterministic_algorithms(True)
    try:
        l1 = torch.stack([s1.step(b, keys[k])[0].clone() for k, b in enumerate(batches)])
        l2 = s2.run(batches, keys)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    s1.sampler.check()
    s2.sampler.check()
    assert torch.isfinite(l1).all()
    assert _same(l1, l2), (l1, l2)
    for a, b in zip(p1, p2):
        assert _same(a, b)


@pytest.mark.parametrize("order", ["step-run-step", "run-step-run"])
def test_step_and_run_mix_in_any_order(order):
    """step(), run(), step() (or run(), step(), run()) on one object: the parameters and losses of the same batches
    through step() alone, with one set of .grad tensors for both entry points."""
    (s1, p1), (s2, p2), n, year = _two_trainers("fp32", 1, None)
    seeds = list(range(70, 77))
    batches = [_seeds(n, year, s) for s in seeds]
    keys = _keys(seeds, 1)
    parts = [(0, 1), (1, 4), (4, 7)]
    torch.use_deterministic_algorithms(True)
    try:
        l1 = torch.stack([s1.step(b, keys[k])[0].clone() for k, b in enumerate(batches)])
        l2, grad_ptrs = [], []
        for i, (a, b) in enumerate(parts):
            if (i % 2 == 0) == order.startswith("step"):
                l2 += [s2.step(batches[k], keys[k])[0].clone() for k in range(a, b)]
            else:
                l2 += list(s2.run(batches[a:b], keys[a:b]))
            grad_ptrs.append([p.grad.data_ptr() for p in p2])
        l2 = torch.stack(l2)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert _same(l1, l2), (l1, l2)
    for a, b in zip(p1, p2):
        assert _same(a, b)
        assert _same(a.grad, b.grad)                       # .grad shows the last call's gradients
    assert all(ptrs == grad_ptrs[0] for ptrs in grad_ptrs)  # the same .grad tensors after step() and run() calls


def _forwards(B):
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = _graphs()
    dg = dgs["fp32"]
    sig = sampler.graph_signature_for(dg, DEPTH, WIDTH, [_seeds(n, year, 5)], 0.5, members=B, time_range=TIME_RANGE)
    gnn, _ = _model(dg, 4)
    gnn.eval()
    fn = lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et)
    out = []
    for _ in range(2):
        gs = sampler.GraphedSampler(dg, sig, DEPTH, WIDTH, {"paper": 128}, members=B, time_range=TIME_RANGE)
        out.append(graphed.GraphedForward(fn, sig, "cuda", sampler=gs))
    return out, n, year


def test_forward_run_hands_consume_the_rows_of_step():
    """members=8 (variance-reduced evaluation): the rows and node_id consume() receives for each batch are bitwise those
    of GraphedForward.step on the same seeds and keys."""
    B = 8
    (f1, f2), n, year = _forwards(B)
    seeds = list(range(80, 85))
    batches = [_seeds(n, year, s) for s in seeds]
    keys = _keys(seeds, B)
    ref = []
    for k, b in enumerate(batches):
        ref.append((f1.step(b, keys[k]), f1.sampler.node_id.clone()))
    got = []
    f2.run(batches, lambda rows, ids: got.append((rows.clone(), ids.clone())), keys)
    torch.cuda.synchronize()
    assert len(got) == len(batches)
    for (r1, i1), (r2, i2) in zip(ref, got):
        assert _same(r1, r2)
        assert torch.equal(i1, i2)
        assert int((i1 >= 0).sum()) > 0


def test_run_does_not_synchronise():
    (s1, _), _, n, year = _two_trainers("fp32", 1, None)
    (f1, _), _, _ = _forwards(2)
    batches = [_seeds(n, year, s) for s in range(90, 94)]
    keys = _keys(range(4), 1)
    s1.run(batches[:2])                                    # first calls: capture
    s1.step(batches[0])
    f1.run(batches[:2], lambda rows, ids: None)
    torch.cuda.synchronize()
    kept = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = s1.run(batches)
        f1.run(batches, lambda rows, ids: kept.append(rows.sum()))
        s1.step(batches[0])
        losses2 = s1.run(batches, keys)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(losses).all() and torch.isfinite(losses2).all()
    assert len(kept) == len(batches) and all(bool(torch.isfinite(v)) for v in kept)


def _sizes(dg, sig_loose, batches, keys, B):
    """Exact per-type node counts and edge counts of each batch, from a GraphedSampler on a loose signature."""
    from pyhgt_b200 import sampler
    gs = sampler.GraphedSampler(dg, sig_loose, DEPTH, WIDTH, {"paper": 128}, members=B, time_range=TIME_RANGE)
    out = []
    for k, b in enumerate(batches):
        gs.fill(b, keys[k])
        gs.check()
        real = gs.node_id >= 0
        counts = [int((real & (gs.nt == t)).sum()) for t in range(len(dg.types))]
        out.append((counts, int(gs.n_real)))
    return out


def test_a_bad_batch_in_the_list():
    """A batch past the signature in the middle of a run: the losses are those of the same step() calls (NaN from that
    batch on, since its NaN update reaches the parameters), the forward's rows are NaN for that batch only, and
    check() names its index."""
    from pyhgt_b200 import graphed, sampler
    dgs, n, year = _graphs()
    dg = dgs["fp32"]
    seeds = list(range(100, 106))
    batches = [_seeds(n, year, s, count=16) for s in seeds]
    bad = 3
    batches[bad] = _seeds(n, year, seeds[bad], count=128)
    keys = _keys(seeds, 1)
    loose = sampler.graph_signature_for(dg, DEPTH, WIDTH, [_seeds(n, year, 1)], 3.0, time_range=TIME_RANGE)
    sizes = _sizes(dg, loose, batches, keys, 1)
    good = [s for k, s in enumerate(sizes) if k != bad]
    counts = [max(c[t] for c, _ in good) for t in range(len(dg.types))]
    edges = max(e for _, e in good)
    assert any(c > m for c, m in zip(sizes[bad][0], counts)) or sizes[bad][1] > edges
    sig = graphed.GraphSignature(counts, edges, sampler._mag_pairs(dg), len(dg.edge_dict), dg.feat_dim)

    (s1, p1), (s2, p2), _, _ = _two_trainers("fp32", 1, None, sig=sig)
    torch.use_deterministic_algorithms(True)
    try:
        l1 = torch.stack([s1.step(b, keys[k])[0].clone() for k, b in enumerate(batches)])
        l2 = s2.run(batches, keys)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.isfinite(l1[:bad]).all() and torch.isnan(l1[bad:]).all()
    assert _same(l1, l2), (l1, l2)
    for a, b in zip(p1, p2):
        assert _same(a, b)
    with pytest.raises(ValueError, match="^seed batch %d: " % bad):
        s2.sampler.check()

    gnn, _ = _model(dg, 4)
    gnn.eval()
    gs = sampler.GraphedSampler(dg, sig, DEPTH, WIDTH, {"paper": 128}, time_range=TIME_RANGE)
    fwd = graphed.GraphedForward(lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et), sig, "cuda", sampler=gs)
    rows = []
    fwd.run(batches, lambda r, ids: rows.append((r.clone(), ids.clone())), keys)
    torch.cuda.synchronize()
    for k, (r, ids) in enumerate(rows):
        if k == bad:               # nothing laid out, every feature NaN: every row but the closing out-of-type node's
            assert int((ids >= 0).sum()) == 0 and bool(torch.isnan(r[:sig.n_nodes - 1]).all()), k
        else:
            assert int((ids >= 0).sum()) > 0 and bool(torch.isfinite(r[ids >= 0]).all()), k
    with pytest.raises(ValueError, match="^seed batch %d: " % bad):
        gs.check()
