"""sampler.sample_subgraph_cuda (HGSampling + to_torch on the GPU) against the host sampler, which replays the
reference's numpy stream bit for bit (tests/test_sampler.py):

  * given the sampled nodes, the device rebuild and layout equal the host `_finish` + `to_torch` bitwise;
  * over many seeds, both draw the same distribution of sampled nodes, their times and the batch sizes;
  * the same generator seed gives bitwise-identical batches;
  * edge cases of the budget process, and a training loop driven by device batches."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import load_golden          # noqa: E402
from tests.test_sampler import _GraphStub, _extractor   # noqa: E402

M = 2000          # samples per side in the distribution test


def _dev():
    return torch.device("cuda:0")


def _tables(fg, types, width=8, seed=0):
    rng = np.random.RandomState(seed)
    return {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 0), 1), width).astype(np.float32)) for t in types}


def _device_graph(name, features=True):
    from pyhgt_b200 import sampler
    fx = load_golden(name)
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types()) if features else None
    return fx, g, fg, sampler.DeviceGraph(fg, _dev(), tabs), tabs


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _host_rebuild(fg, g, tabs, indxs, node_time):
    """Host _finish + to_torch on the node state the device sampled."""
    from pyhgt_b200 import data as hdata, sampler
    states = {}
    for t, ids in indxs.items():
        ids = ids.cpu().numpy()
        tms = node_time[t].cpu().numpy()
        st = sampler._TypeState(max(fg.n_ids.get(t, 0), int(ids.max()) + 1))
        st.layer_ids = ids.tolist()
        st.ser[ids] = np.arange(ids.shape[0])
        st.in_layer[ids] = True
        st.layer_time[ids] = tms
        states[t] = st

    def extractor(layer_data, graph):
        feature, times, ind = {}, {}, {}
        for t in g.get_types():
            ids = np.array(list(layer_data[t].keys()), dtype=np.int64) if t in layer_data else np.zeros(0, np.int64)
            feature[t] = tabs[t].numpy()[ids] if tabs is not None else np.zeros((ids.shape[0], 1), np.float32)
            times[t] = np.array([layer_data[t][i][1] for i in ids], dtype=np.int64)
            ind[t] = ids
        return feature, times, ind, []

    feature, times, edge_list, _, _ = sampler._finish(fg, states, list(indxs.keys()), extractor)
    return hdata.to_torch(feature, times, edge_list, g)


def _assert_same_as_host_rebuild(out, fg, g, tabs):
    ref = _host_rebuild(fg, g, tabs, out[7], out[8])
    if tabs is not None:
        assert torch.equal(out[0].cpu(), ref[0])
    for i in (1, 2, 3, 4):
        assert torch.equal(out[i].cpu(), ref[i]), i
    assert out[5] == ref[5] and out[6] == ref[6]


@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
def test_device_rebuild_equals_host_finish_and_to_torch(name):
    from pyhgt_b200 import sampler
    fx, g, fg, dg, tabs = _device_graph(name)
    for case in fx["cases"]:
        for seed in range(3):
            out = sampler.sample_subgraph_cuda(dg, fx["time_range"], case["depth"], case["number"], fx["inp"], _gen(seed))
            _assert_same_as_host_rebuild(out, fg, g, tabs)
            # seeds are the first nodes of their type, in inp order (data.py:135-137)
            for t, arr in fx["inp"].items():
                n = len(arr)
                assert out[7][t][:n].cpu().tolist() == [int(a[0]) for a in arr]


# ---- same distribution ---------------------------------------------------------------------------------

def host_stats(name, depth, width, m=M):
    from pyhgt_b200 import sampler
    fx = load_golden(name)
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    incl, timed, sizes, edges = {}, {}, {t: [] for t in g.get_types()}, []
    for i in range(m):
        np.random.seed(i)
        _, times, edge_list, indxs, _ = sampler.sample_subgraph(fg, fx["time_range"], depth, width, fx["inp"], _extractor)
        _accumulate(incl, timed, sizes, g.get_types(), {t: (np.asarray(indxs[t]), np.asarray(times[t])) for t in indxs})
        edges.append(sum(len(edge_list[a][b][c]) for a in edge_list for b in edge_list[a] for c in edge_list[a][b]))
    return incl, timed, sizes, edges


def device_stats(name, depth, width, m=M):
    from pyhgt_b200 import sampler
    fx, g, fg, dg, _ = _device_graph(name, features=False)
    incl, timed, sizes, edges = {}, {}, {t: [] for t in g.get_types()}, []
    for i in range(m):
        out = sampler.sample_subgraph_cuda(dg, fx["time_range"], depth, width, fx["inp"], _gen(i))
        _accumulate(incl, timed, sizes, g.get_types(),
                    {t: (out[7][t].cpu().numpy(), out[8][t].cpu().numpy()) for t in out[7]})
        edges.append(int(out[3].shape[1]))
    return incl, timed, sizes, edges


def _accumulate(incl, timed, sizes, types, got):
    for t in types:
        ids, tms = got.get(t, (np.zeros(0, np.int64), np.zeros(0, np.int64)))
        sizes[t].append(len(ids))
        for i, tm in zip(ids.tolist(), tms.tolist()):
            incl[(t, i)] = incl.get((t, i), 0) + 1
            timed[(t, i, tm)] = timed.get((t, i, tm), 0) + 1


def compare_stats(h, d, m=M):
    """Failures of the frequency bound and of the chi-square tests (empty list = same distribution)."""
    from scipy.stats import chi2_contingency
    bad = []
    for which, (ch, cd) in (("inclusion", (h[0], d[0])), ("node/time", (h[1], d[1]))):
        for key in set(ch) | set(cd):
            a, b = ch.get(key, 0) / m, cd.get(key, 0) / m
            p = (a + b) / 2
            if 0.02 <= p <= 0.98 and abs(a - b) > 5 * np.sqrt(2 * p * (1 - p) / m):
                bad.append((which, key, a, b))
    hists = [("nodes of %s" % t, h[2][t], d[2][t]) for t in h[2]] + [("edges", h[3], d[3])]
    for label, xs, ys in hists:
        vals = np.array(sorted(set(xs) | set(ys)))
        if vals.shape[0] < 2:
            if list(xs) != list(ys):
                bad.append((label, "support", None, None))
            continue
        # bins of at least 5 expected per side: cut the sorted support where the pooled count reaches 10
        pooled = np.concatenate([xs, ys])
        cuts, acc = [], 0
        for v in vals:
            acc += int(np.sum(pooled == v))
            if acc >= 10:
                cuts.append(v)
                acc = 0
        if not cuts:
            continue
        cuts[-1] = vals[-1]
        edges_ = np.concatenate([[vals[0] - 1], cuts])
        table = np.array([np.histogram(xs, edges_ + 0.5)[0], np.histogram(ys, edges_ + 0.5)[0]])
        table = table[:, table.sum(0) > 0]
        if table.shape[1] < 2:
            continue
        pval = chi2_contingency(table)[1]
        if pval <= 1e-4:
            bad.append((label, "chi2", pval, None))
    return bad


_CASES = [("sampler", 2, 8), ("sampler", 4, 16), ("sampler_large", 5, 64)]


@pytest.mark.parametrize("name,depth,width", _CASES)
def test_device_sampler_draws_the_host_distribution(name, depth, width):
    fx = load_golden(name)
    assert (depth, width) in [(c["depth"], c["number"]) for c in fx["cases"]]
    bad = compare_stats(host_stats(name, depth, width), device_stats(name, depth, width))
    assert not bad, bad[:10]


# ---- reproducibility -----------------------------------------------------------------------------------

def _equal_outputs(a, b):
    for i in range(5):
        if (a[i] is None) != (b[i] is None) or (a[i] is not None and not torch.equal(a[i], b[i])):
            return False
    return (a[5] == b[5] and list(a[7]) == list(b[7]) and
            all(torch.equal(a[7][t], b[7][t]) and torch.equal(a[8][t], b[8][t]) for t in a[7]))


def test_same_seed_same_batch_other_seed_other_batch():
    from pyhgt_b200 import sampler
    fx, g, fg, dg, _ = _device_graph("sampler_large")
    c = fx["cases"][0]
    run = lambda s: sampler.sample_subgraph_cuda(dg, fx["time_range"], c["depth"], c["number"], fx["inp"], _gen(s))
    a, b, other = run(5), run(5), run(6)
    assert _equal_outputs(a, b)
    assert not _equal_outputs(a, other)


# ---- edge cases ----------------------------------------------------------------------------------------

def test_seed_ids_beyond_the_graph_and_a_seed_type_without_edges():
    from pyhgt_b200 import sampler
    fx = load_golden("sampler")
    g = _GraphStub(fx)
    g._t = g._t + ["never_seen_type"]
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types())
    big = max(fg.n_ids.values()) + 7
    tabs["paper"] = torch.randn(big + 1, 8)
    tabs["never_seen_type"] = torch.randn(4, 8)
    dg = sampler.DeviceGraph(fg, _dev(), tabs)
    first = next(iter(fx["inp"]))
    seeds = np.concatenate([np.asarray(fx["inp"][first]), [[big, 2010]]])
    out = sampler.sample_subgraph_cuda(dg, fx["time_range"], 2, 8, {first: seeds, "never_seen_type": np.array([[3, 2011]])},
                                       _gen(0))
    assert big in out[7][first].cpu().tolist() and out[7]["never_seen_type"].cpu().tolist() == [3]
    _assert_same_as_host_rebuild(out, fg, g, tabs)
    # both are isolated: their only edge is the self loop
    row = out[5]["never_seen_type"][0]
    ei = out[3].cpu()
    assert ((ei[0] == row) | (ei[1] == row)).sum() == 1
    with pytest.raises(KeyError):
        sampler.sample_subgraph_cuda(dg, fx["time_range"], 2, 8, {"not_a_type": np.array([[0, 2010]])}, _gen(0))


class _Stub:
    def __init__(self, edge_list, types, meta):
        self.edge_list, self._t, self._m = edge_list, types, meta

    def get_types(self):
        return self._t

    def get_meta_graph(self):
        return self._m


def _small(adj):
    """paper <- author graph: adj[paper] = [author, ...] (edge time 2000), plus the reverse block."""
    from collections import defaultdict
    el = defaultdict(lambda: defaultdict(lambda: defaultdict(dict)))
    for p, authors in adj.items():
        for a in authors:
            el["paper"]["author"]["AP_write"].setdefault(p, {})[a] = 2000
            el["author"]["paper"]["rev_AP_write"].setdefault(a, {})[p] = 2000
    return _Stub(el, ["paper", "author"], [("paper", "author", "AP_write"), ("author", "paper", "rev_AP_write")])


def test_budget_smaller_than_and_equal_to_the_width():
    """Budget a0: 1/4 + 1/2, a1..a3: 1/4, a4: 1/2 (five entries, inserted a0..a4).  Width 6 takes all of them in
    insertion order; width 5 == budget size samples them all with p ~ score^2, so a0 comes first with probability
    0.5625 / (0.5625 + 3 * 0.0625 + 0.25)."""
    from pyhgt_b200 import sampler
    g = _small({0: [10, 11, 12, 13], 1: [10, 14]})
    dg = sampler.DeviceGraph(sampler.FrozenGraph(g), _dev())
    inp = {"paper": np.array([[0, 2000], [1, 2000]])}
    for s in range(20):
        out = sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 6, inp, _gen(s))
        assert out[7]["author"].cpu().tolist() == [10, 11, 12, 13, 14]
    firsts, orders = [], set()
    n = 400
    for s in range(n):
        out = sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 5, inp, _gen(s))
        got = out[7]["author"].cpu().tolist()
        assert sorted(got) == [10, 11, 12, 13, 14]
        firsts.append(got[0])
        orders.add(tuple(got))
    p = 0.5625
    assert abs(np.mean(np.array(firsts) == 10) - p) < 5 * np.sqrt(p * (1 - p) / n)
    assert len(orders) > 10


def test_target_with_degree_far_above_the_width():
    """A seed with 4000 neighbours and width 8: an ordered uniform 8-subset per batch (all of it is then sampled)."""
    from scipy.stats import chisquare
    from pyhgt_b200 import sampler
    deg = 4000
    g = _small({0: list(range(deg))})
    dg = sampler.DeviceGraph(sampler.FrozenGraph(g), _dev())
    inp = {"paper": np.array([[0, 2000]])}
    draws, firsts = [], []
    for s in range(400):
        got = sampler.sample_subgraph_cuda(dg, {2000: True}, 1, 8, inp, _gen(s))[7]["author"].cpu().numpy()
        assert got.shape[0] == 8 and np.unique(got).shape[0] == 8 and got.min() >= 0 and got.max() < deg
        draws.append(got)
        firsts.append(got[0])
    draws = np.concatenate(draws)
    assert chisquare(np.histogram(draws, 16, (0, deg))[0]).pvalue > 1e-4
    assert chisquare(np.histogram(firsts, 8, (0, deg))[0]).pvalue > 1e-4


def test_time_range_none_disables_the_time_filter():
    from pyhgt_b200 import sampler
    fx, g, fg, dg, _ = _device_graph("sampler", features=False)
    max_t = max(fx["time_range"])
    seen_late = False
    for s in range(5):
        off = sampler.sample_subgraph_cuda(dg, None, 4, 16, fx["inp"], _gen(s))
        huge = sampler.sample_subgraph_cuda(dg, {10 ** 9: True}, 4, 16, fx["inp"], _gen(s))
        assert _equal_outputs(off, huge)              # no filter == a filter that never fires
        on = sampler.sample_subgraph_cuda(dg, fx["time_range"], 4, 16, fx["inp"], _gen(s))
        for t in on[8]:
            n_seed = len(fx["inp"].get(t, []))
            if on[8][t].numel() > n_seed:                     # sampled (non-seed) nodes pass the filter
                assert int(on[8][t][n_seed:].max()) <= max_t
        seen_late |= any(int(off[8][t].max()) > max_t for t in off[8])
    assert seen_late


def test_duplicate_seeds_raise():
    from pyhgt_b200 import sampler
    fx, g, fg, dg, _ = _device_graph("sampler", features=False)
    with pytest.raises(ValueError):
        sampler.sample_subgraph_cuda(dg, fx["time_range"], 2, 8, {"paper": np.array([[1, 2010], [1, 2011]])}, _gen(0))


# ---- integration ---------------------------------------------------------------------------------------

def test_device_sampled_minibatch_training_reduces_the_loss():
    """tests/test_gpu_training_loop.py with the device sampler; the forward passes run with host syncs forbidden."""
    from pyhgt_b200 import sampler
    from pyhgt_b200.model import GNN
    import pyhgt_b200
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
    dg = sampler.DeviceGraph(fg, dev, {t: torch.from_numpy(v) for t, v in table.items()})

    years = {}
    for a, papers in fx["edge_list"]["paper"]["author"]["AP_write"].items():
        for _author, t in papers.items():
            years[a] = t
    labelled = np.array([p for p in range(n_paper) if venue_of[p] >= 0 and p in years])
    edge_dict = {e[2]: i for i, e in enumerate(g.get_meta_graph())}
    edge_dict["self"] = len(edge_dict)
    torch.manual_seed(0)
    gnn = GNN(F_in, n_hid, len(types), len(edge_dict), 4, 2, 0.0, "hgt", True, False, True).to(dev).train()
    head = torch.nn.Linear(n_hid, n_cls).to(dev)
    opt = torch.optim.Adam(list(gnn.parameters()) + list(head.parameters()), lr=2e-3)
    old_keep = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = False
    losses = []
    gen = _gen(0)
    try:
        for step in range(40):
            np.random.seed(step)
            batch = np.random.choice(labelled, 32, replace=False)
            inp = {"paper": np.array([[int(p), int(years[p])] for p in batch])}
            nf, nt, etime, ei, et, node_dict, _, _, _ = sampler.sample_subgraph_cuda(dg, fx["time_range"], 3, 12, inp, gen)
            labels = torch.from_numpy(venue_of[batch]).to(dev)
            # step 0 uploads the layers' parameter pointer tables (a one-time copy); every later forward is sync-free
            torch.cuda.set_sync_debug_mode("error" if step else 0)
            try:
                out = gnn(nf, nt, etime, ei, et)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            p0 = node_dict["paper"][0]
            logits = head(out[p0:p0 + len(batch)])
            loss = torch.nn.functional.cross_entropy(logits, labels)
            opt.zero_grad()
            loss.backward()
            for name, p in gnn.named_parameters():
                assert p.grad is None or torch.isfinite(p.grad).all(), name
            opt.step()
            losses.append(float(loss))
    finally:
        pyhgt_b200.HGTConv.keep_att = old_keep
    assert np.isfinite(losses).all()
    assert np.mean(losses[-8:]) < 0.7 * np.mean(losses[:8]), losses
