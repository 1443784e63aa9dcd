"""sampler.sample_subgraphs_cuda (B subgraphs in one device pass) and sampler.merge_batches (their disjoint union):

  * member b of a batched call is bitwise sample_subgraph_cuda from a generator advanced by b draws, in all nine
    outputs (which, with the single path's distribution test, is also the batched path's distribution guarantee);
  * a batched call synchronises depth + 1 times whatever B is;
  * GNN / HGTConv on the union give every member's rows as on the member alone, with no host synchronisation."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import load_golden                    # noqa: E402
from tests.test_gpu_sampler import _dev, _gen, _small, _tables   # noqa: E402
from tests.test_sampler import _GraphStub                 # noqa: E402


def _graph(name):
    """The fixture graph plus a node type without edges; paper features reach past the id range."""
    from pyhgt_b200 import sampler
    fx = load_golden(name)
    g = _GraphStub(fx)
    g._t = g._t + ["never_seen_type"]
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types())
    big = max(fg.n_ids.values()) + 7
    tabs["paper"] = torch.randn(big + 1, 8)
    tabs["never_seen_type"] = torch.randn(4, 8)
    return fx, fg, sampler.DeviceGraph(fg, _dev(), tabs), big


def _inps(fx, fg, big, B, seed=0):
    """B seed dicts: the fixture's seeds (identical members, as in variance-reduced evaluation), other paper seeds, seeds
    beyond the id range plus a seed type without edges, and members whose seeds start from other types."""
    rng = np.random.RandomState(seed)
    out = []
    for b in range(B):
        kind = b % 5
        if kind == 0:
            inp = fx["inp"]
        elif kind == 1:
            ids = rng.choice(fg.n_ids["paper"], 16, replace=False)
            inp = {"paper": np.stack([ids, rng.randint(2000, 2016, 16)], 1)}
        elif kind == 2:
            inp = {"paper": np.concatenate([np.asarray(fx["inp"]["paper"]), [[big, 2010]]]),
                   "never_seen_type": np.array([[3, 2011]])}
        elif kind == 3:
            a = rng.choice(fg.n_ids["author"], 8, replace=False)
            p = rng.choice(fg.n_ids["paper"], 4, replace=False)
            inp = {"author": np.stack([a, np.full(8, 2005)], 1), "paper": np.stack([p, np.full(4, 2012)], 1)}
        else:
            f = rng.choice(fg.n_ids["field"], 3, replace=False)
            inp = {"field": np.stack([f, np.full(3, 2008)], 1)}
        out.append(inp)
    return out


def _assert_bitwise(a, b):
    for i in range(5):
        assert (a[i] is None) == (b[i] is None), i
        if a[i] is not None:
            assert a[i].shape == b[i].shape and torch.equal(a[i], b[i]), i
    assert a[3].is_contiguous()
    assert a[5] == b[5] and a[6] == b[6]
    assert list(a[7]) == list(b[7]) and list(a[8]) == list(b[8])
    for t in a[7]:
        assert torch.equal(a[7][t], b[7][t]) and torch.equal(a[8][t], b[8][t]), t


def _singles(dg, time_range, depth, width, inps, seed):
    """sample_subgraph_cuda of every seed dict, member b from the generator advanced by b draws."""
    from pyhgt_b200 import sampler
    out = []
    for b, inp in enumerate(inps):
        g = _gen(seed)
        for _ in range(b):
            torch.randint(0, 2 ** 63 - 1, (1,), generator=g)
        out.append(sampler.sample_subgraph_cuda(dg, time_range, depth, width, inp, g))
    return out


@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("depth,width", [(2, 8), (5, 64)])
@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
def test_member_b_is_the_single_call_with_the_generator_advanced_b_draws(name, depth, width, B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph(name)
    inps = _inps(fx, fg, big, B)
    got = sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, width, inps, _gen(11))
    assert len(got) == B
    ref = _singles(dg, fx["time_range"], depth, width, inps, 11)
    for b in range(B):
        _assert_bitwise(got[b], ref[b])
    if B >= 5:
        # members walk their types in different orders (the per-member type array is exercised), and the seeds beyond
        # the id range and of the type without edges are sampled
        assert len({tuple(o[7]) for o in got}) >= 2
        assert big in got[2][7]["paper"].cpu().tolist() and got[2][7]["never_seen_type"].cpu().tolist() == [3]


def test_identical_seeds_draw_independent_members():
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    got = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 5, 64, [fx["inp"]] * 4, _gen(3))
    assert len({tuple(o[7]["paper"].cpu().tolist()) for o in got}) == 4


@pytest.mark.parametrize("B", [1, 5])
def test_time_range_none(B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler")
    inps = _inps(fx, fg, big, B, seed=1)
    got = sampler.sample_subgraphs_cuda(dg, None, 4, 16, inps, _gen(2))
    ref = _singles(dg, None, 4, 16, inps, 2)
    for b in range(B):
        _assert_bitwise(got[b], ref[b])


def test_budget_smaller_than_the_width():
    """Width 6 over a five-entry budget takes all of it in insertion order (test_gpu_sampler.py); width 5 samples it."""
    from pyhgt_b200 import sampler
    g = _small({0: [10, 11, 12, 13], 1: [10, 14]})
    dg = sampler.DeviceGraph(sampler.FrozenGraph(g), _dev())
    inps = [{"paper": np.array([[0, 2000], [1, 2000]])}, {"paper": np.array([[1, 2000]])},
            {"author": np.array([[10, 2000]])}]
    for width in (6, 5):
        got = sampler.sample_subgraphs_cuda(dg, {2000: True}, 1, width, inps, _gen(width))
        ref = _singles(dg, {2000: True}, 1, width, inps, width)
        for b in range(3):
            _assert_bitwise(got[b], ref[b])
        if width == 6:
            assert got[0][7]["author"].cpu().tolist() == [10, 11, 12, 13, 14]


def test_errors_are_per_member_and_keep_their_messages():
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler")
    with pytest.raises(ValueError, match="duplicate seed ids"):
        sampler.sample_subgraphs_cuda(dg, fx["time_range"], 2, 8, [fx["inp"], {"paper": np.array([[1, 2010], [1, 2011]])}])
    with pytest.raises(KeyError):
        sampler.sample_subgraphs_cuda(dg, fx["time_range"], 2, 8, [fx["inp"], {"not_a_type": np.array([[0, 2010]])}])
    assert sampler.sample_subgraphs_cuda(dg, fx["time_range"], 2, 8, []) == []


@pytest.mark.parametrize("B", [1, 8, 32])
def test_host_syncs_are_depth_plus_one_for_every_B(B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    inps = _inps(fx, fg, big, B)
    depth = 5
    sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, 64, inps, _gen(0))        # warm-up
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, 64, inps, _gen(1))
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [x for x in w if str(x.message).startswith("called a synchronizing CUDA operation")]
    assert len(syncs) == depth + 1, [str(x.message) for x in syncs]


# ---- disjoint union --------------------------------------------------------------------------------------------------

def _modules(T, R, F):
    import pyhgt_b200
    from pyhgt_b200.model import GNN
    torch.manual_seed(0)
    gnn = GNN(F, 32, T, R, 4, 2, 0.0, "hgt", True, False, True).to(_dev()).eval()
    conv = pyhgt_b200.HGTConv(32, 32, T, R, 4, 0.0, True, True).to(_dev()).eval()
    return gnn, conv


def _check_union(batches, T, R, F):
    from pyhgt_b200 import sampler
    gnn, conv = _modules(T, R, F)
    wide = lambda x: x.repeat(1, 32 // F)                    # the bare layer needs in_dim == out_dim (skip connection)
    with torch.no_grad():
        alone = [(gnn(*m[:5]), conv(wide(m[0]), m[1], m[3], m[4], m[2])) for m in batches]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            nf, nt, etime, ei, et, rows = sampler.merge_batches(batches, T, R)
            y_gnn = gnn(nf, nt, etime, ei, et)
            y_conv = conv(wide(nf), nt, ei, et, etime)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert bool((nt[1:] >= nt[:-1]).all())
    assert nt.numel() == sum(m[1].numel() for m in batches) and ei.shape[1] == sum(m[3].shape[1] for m in batches)
    worst, bitwise = 0.0, True
    for b, m in enumerate(batches):
        assert torch.equal(nt[rows[b]], m[1]) and torch.equal(nf[rows[b]], m[0])
        for u, a in ((y_gnn, alone[b][0]), (y_conv, alone[b][1])):
            d = (u[rows[b]] - a).abs().max().item() if a.numel() else 0.0
            worst = max(worst, d)
            bitwise &= torch.equal(u[rows[b]], a)
    assert worst <= 1e-5, worst
    return bitwise


@pytest.mark.parametrize("B", [1, 5])
def test_union_forward_gives_every_members_rows(B):
    from pyhgt_b200 import sampler
    fx, fg, dg, big = _graph("sampler_large")
    batches = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 32, _inps(fx, fg, big, B), _gen(4))
    bitwise = _check_union(batches, len(dg.types), len(dg.edge_dict), dg.feat_dim)
    print("union rows bitwise equal to the members' own forward: %s" % bitwise)


def test_union_of_members_with_disjoint_relation_pairs():
    from pyhgt_b200 import sampler
    g = _small({0: [10, 11, 12, 13], 1: [10, 14]})
    fg = sampler.FrozenGraph(g)
    dg = sampler.DeviceGraph(fg, _dev(), _tables(fg, g.get_types()))
    # depth 0: only the seeds and their self loops, so the <type, relation> pairs are {paper-self} and {author-self}
    batches = sampler.sample_subgraphs_cuda(dg, {2000: True}, 0, 4, [{"paper": np.array([[0, 2000], [1, 2000]])},
                                                                      {"author": np.array([[10, 2000], [14, 2000]])}],
                                            _gen(0))
    from pyhgt_b200 import plan as _plan
    T, R = len(dg.types), len(dg.edge_dict)
    p = [_plan.get_plan(m[1], m[3], m[4], m[2], T, R).pairs for m in batches]
    assert not set(p[0]) & set(p[1])
    _check_union(batches, T, R, dg.feat_dim)
