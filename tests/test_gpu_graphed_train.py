"""graphed.GraphedTrainStep and the capture-safe typed-linear backward on the GPU:

  * hgt_typed_linear_bwd / _det captured alone in a CUDA graph: replays with new operand values equal eager calls;
  * a captured training step (no optimizer) gives the eager loss and gradients on the same padded inputs bitwise under
    the deterministic flag, and the unpadded batch's within 1e-5;
  * the ogbn-mag recipe (AdamW capturable + tensor lr, OneCycleLR, clip 1.0): 10 graphed calls = 10 eager steps;
  * device batches from sample_subgraphs_cuda feed both graphed classes with no host synchronisation;
  * a graphed sampled-minibatch task with dropout learns; misfit batches, new pairs, non-capturable optimizers and a
    flag change after capture are refused."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pyhgt_b200 import graphed, synth  # noqa: E402


def _dev():
    return torch.device("cuda:0")


class _Det:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(self.on, warn_only=True)

    def __exit__(self, *a):
        torch.use_deterministic_algorithms(self.old)


@pytest.fixture(autouse=True)
def _no_att():
    import pyhgt_b200
    old = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = False
    yield
    pyhgt_b200.HGTConv.keep_att = old


def _rel(a, b):
    return (a.double() - b.double()).norm().item() / max(b.double().norm().item(), 1e-30)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the backward GEMM entry points inside a CUDA graph

def _bwd_case(spec, K, width, seed):
    from pyhgt_b200 import plan as P
    dev = _dev()
    gen = torch.Generator().manual_seed(seed)
    groups, cblocks, off, a_row0, w_row0 = [], [], 0, 0, 0
    for gi, (m, nc) in enumerate(spec):
        first = len(cblocks)
        for c in range(nc):
            cblocks.append((off, width))
            off += m * width
        off = (off + 63) // 64 * 64
        groups.append((a_row0, m, w_row0, nc, first, int(gi % 2 == 0)))
        a_row0 += m
        w_row0 += nc * width
    out_elems = off + 64
    tab = P._pack_groups(groups, cblocks, dev)
    W = (torch.randn(w_row0, K, generator=gen) / K ** 0.5).to(dev)
    return tab, len(groups), a_row0, w_row0, out_elems, W, gen


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("impl,spec,dsplit,asplit,gelu,acc", [
    (2, [(300, 3), (129, 1), (64, 2)], True, False, False, False),     # tensor cores, presplit dout, fp32 A
    (2, [(300, 3), (129, 1), (64, 2)], False, True, True, True),       # fp32 dout (split + db), presplit A, gelu, += dA
    (2, [(40 + 7 * g, 7) for g in range(10)], False, False, False, False),   # 70 tasks: the head spans several uploads
    (1, [(300, 3), (129, 1), (64, 2)], False, False, True, True),      # SIMT fp32
    (1, [(40 + 7 * g, 7) for g in range(10)], False, False, False, False),
])
def test_typed_linear_backward_replays_from_a_cuda_graph(det, impl, spec, dsplit, asplit, gelu, acc):
    from pyhgt_b200 import _lib
    K, width = 128, 64
    dev = _dev()
    tab, n_g, rows, w_rows, out_elems, W, gen = _bwd_case(spec, K, width, 5)
    g_dev, g_host, _, _ = tab
    c_host = tab.c_host
    fn = "hgt_typed_linear_bwd_det" if det else "hgt_typed_linear_bwd"
    dout = torch.empty(out_elems, device=dev)
    A = torch.empty(rows, K, device=dev)
    aux = torch.randn(rows, K, generator=gen).to(dev)
    dA0 = torch.randn(rows, K, generator=gen).to(dev)
    d_hi = torch.empty(out_elems, dtype=torch.bfloat16, device=dev) if dsplit else None
    d_lo = torch.empty_like(d_hi) if dsplit else None
    a_hi = torch.empty(rows, K, dtype=torch.bfloat16, device=dev) if asplit else None
    a_lo = torch.empty_like(a_hi) if asplit else None
    dA = torch.empty(rows, K, device=dev)
    dW = torch.empty(w_rows, K, device=dev)
    db = torch.empty(w_rows, device=dev)
    wsb = ctypes.c_size_t()
    _lib.call(fn + "_workspace_bytes", g_host.ctypes.data, n_g, c_host.ctypes.data, K, width, K, out_elems, int(dsplit),
              int(asplit), impl, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)

    def run():
        st = torch.cuda.current_stream().cuda_stream
        dW.zero_()
        db.zero_()
        dA.copy_(dA0)
        if dsplit:
            _lib.call("hgt_act_split", dout.data_ptr(), 64, out_elems // 64, 64, 0, None, d_hi.data_ptr(), d_lo.data_ptr(), st)
        if asplit:
            _lib.call("hgt_act_split", A.data_ptr(), K, rows, K, 0, None, a_hi.data_ptr(), a_lo.data_ptr(), st)
        _lib.call(fn, None if dsplit else dout.data_ptr(), _lib.ptr(d_hi), _lib.ptr(d_lo), out_elems,
                  None if asplit else A.data_ptr(), K, _lib.ptr(a_hi), _lib.ptr(a_lo), W.data_ptr(), K, width,
                  g_dev.data_ptr(), g_host.ctypes.data, n_g, c_host.ctypes.data, dA.data_ptr(), int(acc),
                  aux.data_ptr() if gelu else None, dW.data_ptr(), None if dsplit else db.data_ptr(), impl, ws.data_ptr(),
                  ws.numel(), st)

    def fill(seed):
        g = torch.Generator().manual_seed(seed)
        dout.copy_(torch.randn(out_elems, generator=g))
        A.copy_(torch.randn(rows, K, generator=g))

    fill(0)
    run()                                                   # warm-up (function attributes, driver entry points)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        run()
    for seed in (1, 2):
        fill(seed)
        graph.replay()
        got = [t.clone() for t in (dA, dW, db)]
        run()
        torch.cuda.synchronize()
        for name, a, b in zip(("dA", "dW", "db"), got, (dA, dW, db)):
            assert torch.isfinite(b).all(), name
            if det:
                assert torch.equal(a, b), "%s: graph replay differs from the eager call" % name
            else:
                # the non-deterministic entry point adds dW / db (and the SIMT dA) with float atomics, whose order
                # differs from run to run, eager or graphed
                assert _rel(a, b) < 1e-6, "%s: graph replay vs eager, relative error %.3g" % (name, _rel(a, b))


# ---------------------------------------------------------------------------------------------------------------------
# 2. a captured training step without an optimizer

T, R, F_IN, N_HID, N_CLS = 3, 4, 48, 64, 5


def _batches(seeds=(1, 2, 3)):
    return [synth.make_random(n, e, T, R, seed=s, sorted_types=True, self_loops=20)
            for n, e, s in zip((400, 310, 455, 380), (3000, 2200, 3400, 2900), seeds)]


def _signature(batches, pad=5):
    counts = [max(int((b.node_type == t).sum()) for b in batches) + pad for t in range(T)]
    pairs = {(int(b.node_type[s_]), int(r_)) for b in batches
             for s_, r_ in zip(b.edge_index[0].tolist(), b.edge_type.tolist())}
    return graphed.GraphSignature(counts, max(b.edge_type.numel() for b in batches) + 100, pairs, R, F_IN)


def _features(b):
    return torch.randn(b.num_nodes, F_IN, generator=torch.Generator().manual_seed(7 + b.num_nodes))


def _labels(b):
    n0 = int((b.node_type == 0).sum())
    return torch.randint(0, N_CLS, (n0,), generator=torch.Generator().manual_seed(b.num_nodes))


def _model(kind, use_rte=True, use_norm=True, dropout=0.0):
    from pyhgt_b200.model import GNN
    torch.manual_seed(11)
    gnn = GNN(F_IN, N_HID, T, R, 4, 2, dropout, kind, use_norm, use_norm, use_rte).to(_dev()).train()
    head = torch.nn.Linear(N_HID, N_CLS).to(_dev())
    return gnn, head


def _loss_fn(gnn, head, rows):
    def loss_fn(x, nt, tm, ei, et, targets):
        h = gnn(x, nt, tm, ei, et)[:rows]
        return F.nll_loss(F.log_softmax(head(h), -1), targets[0], ignore_index=-100)
    return loss_fn


@pytest.mark.parametrize("kind,use_rte,use_norm", [("hgt", True, True), ("hgt", False, True), ("hgt", True, False),
                                                   ("dense_hgt", True, True)])
def test_graphed_step_gradients_equal_eager(kind, use_rte, use_norm):
    dev = _dev()
    batches = _batches()
    sig = _signature(batches)
    gnn, head = _model(kind, use_rte, use_norm)
    params = list(gnn.parameters()) + list(head.parameters())
    step = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev, params=params,
                                    targets={0: ((), torch.int64, -100)})
    with _Det(True):
        for rep in range(2):
            for b in batches:
                x, y = _features(b), _labels(b)
                loss, = step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
                torch.cuda.synchronize()
                g_loss = loss.clone()
                static = [p.grad for p in params]
                g_grads = [g.clone() for g in static]
                # eager forward/backward on the same static padded inputs and the same (sync-free) plan
                for p in params:
                    p.grad = None
                step._rebuild_plan()
                ref = step.loss_fn(step.x, step.nt, step.tm, step.ei, step.et, step.y)
                ref.backward()
                assert torch.equal(g_loss, ref.detach()), (kind, rep, b.num_nodes)
                for p, g in zip(params, g_grads):
                    assert torch.equal(g, p.grad), "gradient differs from eager on the padded inputs"
                # eager on the unpadded batch
                for p in params:
                    p.grad = None
                n0 = y.numel()
                out = gnn(x.to(dev), b.node_type.to(dev), b.edge_time.to(dev), b.edge_index.to(dev), b.edge_type.to(dev))
                ref = F.nll_loss(F.log_softmax(head(out[:n0]), -1), y.to(dev))
                ref.backward()
                assert _rel(g_loss, ref.detach()) < 1e-5
                for p, g in zip(params, g_grads):
                    assert _rel(g, p.grad) < 1e-5, "gradient vs the unpadded batch: %.3g" % _rel(g, p.grad)
                for p, g in zip(params, static):
                    p.grad = g


# ---------------------------------------------------------------------------------------------------------------------
# 3. the ogbn-mag recipe: AdamW (capturable, tensor lr), OneCycleLR, clip 1.0

def _recipe(params):
    opt = torch.optim.AdamW(params, lr=torch.tensor(5e-4, device=_dev()), capturable=True)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-3, total_steps=40, pct_start=0.1,
                                                anneal_strategy="linear", final_div_factor=10, cycle_momentum=False)
    return opt, sched


@pytest.mark.parametrize("det", [True, False])
def test_graphed_recipe_matches_eager_steps(det):
    from pyhgt_b200 import plan as P
    dev = _dev()
    batches = _batches() + _batches((4, 5, 6)) + _batches((7, 8, 9)) + _batches((10,))
    sig = _signature(batches)
    gnn, head = _model("hgt")
    gnn2, head2 = copy.deepcopy(gnn), copy.deepcopy(head)
    p1 = list(gnn.parameters()) + list(head.parameters())
    p2 = list(gnn2.parameters()) + list(head2.parameters())
    opt1, sched1 = _recipe(p1)
    opt2, sched2 = _recipe(p2)
    step = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev, optimizer=opt1, clip_norm=1.0,
                                    targets={0: ((), torch.int64, -100)})
    eager_loss = _loss_fn(gnn2, head2, sig.type_counts[0])
    with _Det(det):
        for b in batches[:10]:
            x, y = _features(b), _labels(b)
            step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
            sched1.step()
            # eager: the same padded inputs, the same plan, the same recipe
            px, pnt, ptm, pei, pet, _ = graphed.pad_batch(sig, x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
            tens = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (px, pnt, ptm, pei, pet)]
            tgt = torch.full((sig.type_counts[0],), -100, dtype=torch.int64)
            tgt[:y.numel()] = y
            P.rebuild_plan(tens[1], tens[3], tens[4], tens[2], T, R, sig.host_meta())
            opt2.zero_grad()
            eager_loss(*tens, {0: tgt.to(dev)}).backward()
            torch.nn.utils.clip_grad_norm_(p2, 1.0, foreach=True)
            opt2.step()
            sched2.step()
    torch.cuda.synchronize()
    for a, b in zip(p1, p2):
        if det:
            assert torch.equal(a, b), "parameters differ after 10 steps"
        else:
            assert _rel(a, b) < 1e-5, _rel(a, b)
    for a, b in zip(p1, p2):
        s1, s2 = opt1.state[a], opt2.state[b]
        assert set(s1) == set(s2)
        for k in s1:
            if det:
                assert torch.equal(s1[k], s2[k]), k
            else:
                assert _rel(s1[k], s2[k]) < 1e-5, (k, _rel(s1[k], s2[k]))


# ---------------------------------------------------------------------------------------------------------------------
# 4. device batches from the device sampler

def _device_members(B=4):
    from pyhgt_b200 import sampler
    from tests.test_gpu_sampler import _device_graph, _gen
    fx, g, fg, dg, _ = _device_graph("sampler")
    rng = np.random.RandomState(0)
    inps = [fx["inp"]]
    for _ in range(B - 1):
        ids = rng.choice(fg.n_ids["paper"], 16, replace=False)
        inps.append({"paper": np.stack([ids, rng.randint(2000, 2016, 16)], 1)})
    members = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 8, inps, _gen(3))
    return dg, members


def _device_signature(dg, members):
    from pyhgt_b200 import plan as P
    Td, Rd = len(dg.types), len(dg.edge_dict)
    plans = [P.get_plan(m[1], m[3], m[4], m[2], Td, Rd) for m in members]
    counts = [max(p.type_count[t] for p in plans) + 3 for t in range(Td)]
    pairs = {pr for p in plans for pr in p.pairs}
    return graphed.GraphSignature(counts, max(p.n_edges for p in plans) + 50, pairs, Rd, dg.feat_dim), plans


def test_device_batches_feed_both_graphed_classes_without_host_sync():
    from pyhgt_b200.model import GNN
    dev = _dev()
    dg, members = _device_members()
    sig, plans = _device_signature(dg, members)
    Td, Rd = len(dg.types), len(dg.edge_dict)
    paper = dg.slot["paper"]
    torch.manual_seed(2)
    gnn = GNN(dg.feat_dim, N_HID, Td, Rd, 4, 2, 0.0, "hgt", True, False, True).to(dev)
    head = torch.nn.Linear(N_HID, N_CLS).to(dev)
    params = list(gnn.parameters()) + list(head.parameters())
    # built with the index-less "cuda" while the batches and labels live on cuda:0
    fwd = graphed.GraphedForward(lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et), sig, "cuda")
    r0, C = int(sig.row0[paper]), sig.type_counts[paper]

    def loss_fn(x, nt, tm, ei, et, targets):
        h = gnn(x, nt, tm, ei, et)[r0:r0 + C]
        return F.nll_loss(F.log_softmax(head(h), -1), targets[paper], ignore_index=-100)

    step = graphed.GraphedTrainStep(loss_fn, sig, "cuda", params=params, targets={paper: ((), torch.int64, -100)})
    labels = [torch.randint(0, N_CLS, (p.type_count[paper],), generator=torch.Generator().manual_seed(b)).to(dev)
              for b, p in enumerate(plans)]
    with _Det(True):
        for rep in range(2):
            for b, m in enumerate(members):
                nf, nt, etime, ei, et = m[:5]
                first = fwd.graph is None
                if not first:
                    torch.cuda.set_sync_debug_mode("error")
                try:
                    gnn.eval()
                    out = fwd(nf, nt, etime, ei, et)
                    gnn.train()
                    loss, = step(nf, nt, etime, ei, et, targets={paper: labels[b]})
                finally:
                    torch.cuda.set_sync_debug_mode(0)
                torch.cuda.synchronize()
                # the static inputs equal the host-fed padding
                px, pnt, ptm, pei, pet, _ = graphed.pad_batch(sig, nf.cpu(), nt.cpu(), etime.cpu(), ei.cpu(), et.cpu())
                for g_, h_ in ((step.x, px), (step.nt, pnt), (step.tm, ptm), (step.ei, pei), (step.et, pet),
                               (fwd.x, px), (fwd.ei, pei)):
                    assert np.array_equal(g_.cpu().numpy(), h_)
                # outputs against eager on the member
                gnn.eval()
                with torch.no_grad():
                    ref = gnn(nf, nt, etime, ei, et)
                gnn.train()
                assert (out - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())
                g_loss, g_grads, static = loss.clone(), [p.grad.clone() for p in params], [p.grad for p in params]
                for p in params:
                    p.grad = None
                n_p = labels[b].numel()
                p0 = plans[b].type_row0[paper]
                ref = F.nll_loss(F.log_softmax(head(gnn(nf, nt, etime, ei, et)[p0:p0 + n_p]), -1), labels[b])
                ref.backward()
                assert _rel(g_loss, ref.detach()) < 1e-5
                for p, g in zip(params, g_grads):
                    assert _rel(g, p.grad) < 1e-5
                for p, g in zip(params, static):
                    p.grad = g


# ---------------------------------------------------------------------------------------------------------------------
# 5. a learnable sampled-minibatch task, graphed, with dropout

def test_graphed_sampled_minibatch_training_reduces_the_loss():
    from pyhgt_b200 import data as hdata, sampler
    from pyhgt_b200.model import GNN
    from tests.conftest import load_golden
    from tests.test_sampler import _GraphStub
    dev = _dev()
    fx = load_golden("sampler")
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    types = g.get_types()
    F_in, n_hid = 32, 64
    rng = np.random.RandomState(0)
    n_paper = fg.n_ids["paper"]
    venue_of = np.full(n_paper, -1, dtype=np.int64)
    for v, papers in fx["edge_list"]["venue"]["paper"]["PV_Journal"].items():
        for p in papers:
            venue_of[p] = v
    n_cls = int(venue_of.max()) + 1
    table = {t: rng.randn(fg.n_ids.get(t, 1), F_in).astype(np.float32) * 0.1 for t in types}
    table["paper"][np.arange(n_paper), np.clip(venue_of, 0, None) % F_in] += 1.0

    def extractor(layer_data, graph):
        feature, times, indxs = {}, {}, {}
        for _type in layer_data:
            if len(layer_data[_type]) == 0:
                continue
            idxs = np.array(list(layer_data[_type].keys()))
            feature[_type] = table[_type][idxs]
            times[_type] = np.array(list(layer_data[_type].values()))[:, 1]
            indxs[_type] = idxs
        return feature, times, indxs, []

    years = {}
    for a, papers in fx["edge_list"]["paper"]["author"]["AP_write"].items():
        for _author, t in papers.items():
            years[a] = t
    labelled = np.array([p for p in range(n_paper) if venue_of[p] >= 0 and p in years])
    edge_dict = {e[2]: i for i, e in enumerate(g.get_meta_graph())}
    edge_dict["self"] = len(edge_dict)
    Tn, Rn = len(types), len(edge_dict)
    data = []
    for step_i in range(40):
        np.random.seed(step_i)
        batch = np.random.choice(labelled, 32, replace=False)
        inp = {"paper": np.array([[int(p), int(years[p])] for p in batch])}
        feature, times, edge_list, _, _ = sampler.sample_subgraph(fg, fx["time_range"], 3, 12, inp, extractor)
        tens = hdata.to_torch(feature, times, edge_list, g, device=dev, prebuild_plan=True)
        data.append((tens[:5], torch.from_numpy(venue_of[batch]).to(dev)))
    sig, _ = _device_signature(type("DG", (), {"types": types, "edge_dict": edge_dict, "feat_dim": F_in}),
                               [d[0] for d in data])
    paper = types.index("paper")
    torch.manual_seed(0)
    gnn = GNN(F_in, n_hid, Tn, Rn, 4, 2, 0.2, "hgt", True, False, True).to(dev).train()
    head = torch.nn.Linear(n_hid, n_cls).to(dev)
    opt = torch.optim.Adam(list(gnn.parameters()) + list(head.parameters()), lr=2e-3, capturable=True)
    r0, C = int(sig.row0[paper]), sig.type_counts[paper]

    def loss_fn(x, nt, tm, ei, et, targets):
        return F.cross_entropy(head(gnn(x, nt, tm, ei, et)[r0:r0 + C]), targets[paper], ignore_index=-100)

    step = graphed.GraphedTrainStep(loss_fn, sig, dev, optimizer=opt, targets={paper: ((), torch.int64, -100)})
    losses = []
    for tens, y in data:
        loss, = step(*tens, targets={paper: y})                 # the seed papers are the first papers of the batch
        losses.append(loss.clone())
    losses = torch.stack(losses).cpu().numpy()
    assert np.isfinite(losses).all()
    for p in gnn.parameters():
        assert torch.isfinite(p).all()
    assert np.mean(losses[-8:]) < 0.7 * np.mean(losses[:8]), losses


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals

def test_graphed_step_refusals():
    dev = _dev()
    batches = _batches()
    sig = _signature(batches)
    gnn, head = _model("hgt")
    params = list(gnn.parameters()) + list(head.parameters())
    with pytest.raises(ValueError, match="capturable"):
        graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev,
                                 optimizer=torch.optim.AdamW(params, lr=1e-3))
    opt = torch.optim.AdamW(params, lr=1e-3, capturable=True)
    step = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev, optimizer=opt,
                                    targets={0: ((), torch.int64, -100)})
    b = batches[0]
    x, y = _features(b), _labels(b)
    with _Det(False):
        step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
        torch.cuda.synchronize()
        before = [p.detach().clone() for p in params]
        big = synth.make_random(2000, 3000, T, R, seed=9, sorted_types=True)
        with pytest.raises(ValueError):                                            # more nodes than the signature
            step(torch.randn(2000, F_IN), big.node_type, big.edge_time, big.edge_index, big.edge_type,
                 targets={0: _labels(big)[:10]})
        with pytest.raises(ValueError):                                            # labels for more rows than nodes
            step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type,
                 targets={0: torch.zeros(sig.type_counts[0] + 1, dtype=torch.int64)})
        # a <source type, relation> pair the signature does not have: a signature without one of b's pairs, captured on b
        # minus that pair's edges, refuses b itself, from the host and from the device, in both graphed classes
        drop = (int(b.node_type[b.edge_index[0, 0]]), int(b.edge_type[0]))
        sig_less = graphed.GraphSignature(sig.type_counts, sig.n_edges, [pr for pr in sig.pairs if pr != drop], R, F_IN)
        keep = ~((b.node_type[b.edge_index[0]] == drop[0]) & (b.edge_type == drop[1]))
        step_less = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig_less, dev, params=params,
                                             targets={0: ((), torch.int64, -100)})
        fwd_less = graphed.GraphedForward(lambda *a: gnn(*a), sig_less, dev)
        step_less(x, b.node_type, b.edge_time[keep], b.edge_index[:, keep], b.edge_type[keep], targets={0: y})
        with torch.no_grad():
            fwd_less(x, b.node_type, b.edge_time[keep], b.edge_index[:, keep], b.edge_type[keep])
        host = (x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
        device = tuple(t.to(dev) for t in host)
        for batch in (host, device):
            with pytest.raises(ValueError, match="pairs"):
                step_less(*batch, targets={0: y})
            with pytest.raises(ValueError, match="pairs"):
                fwd_less(*batch)
        torch.cuda.synchronize()
        for p, q in zip(params, before):                                          # nothing ran
            assert torch.equal(p, q)
    with _Det(True):
        with pytest.raises(RuntimeError, match="deterministic"):
            step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
    # a hyperparameter the graph holds by value (OneCycleLR cycles AdamW's betas by default) must not change
    opt = torch.optim.AdamW(params, lr=torch.tensor(1e-3, device=dev), capturable=True)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-3, total_steps=40, pct_start=0.1)
    step = graphed.GraphedTrainStep(_loss_fn(gnn, head, sig.type_counts[0]), sig, dev, optimizer=opt,
                                    targets={0: ((), torch.int64, -100)})
    step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
    sched.step()
    with pytest.raises(RuntimeError, match="betas"):
        step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
