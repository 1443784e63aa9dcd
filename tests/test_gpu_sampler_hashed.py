"""sample_subgraphs_cuda on the hashed sampler state (per (member, type) hash tables sized by the sample):

  * every batch is bitwise the dense state's, with the same cached plan, across fixtures, B, the time filter, the OAG
    edge masks, device and host placement, with and without features, and for a hub far above the width;
  * a region too small for the sample overflows, the call restarts from the same draws with a grown room and still
    gives the dense batch, and the next call fits;
  * a seed id past 2^31 (which the dense state cannot sort) samples, and ids from 2^40 on are refused."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.test_gpu_sampler import _dev, _gen, _small, _tables   # noqa: E402
from tests.test_gpu_sampler_batched import _assert_bitwise, _inps   # noqa: E402
from tests.test_gpu_sampler_host import _pair               # noqa: E402
from tests.test_gpu_sampler_mask import _rules              # noqa: E402


def _as(layout, fn, monkeypatch):
    from pyhgt_b200 import sampler
    with monkeypatch.context() as m:
        m.setattr(sampler, "_FORCE_LAYOUT", layout)
        return fn()


def _assert_same(a, b, dg):
    from pyhgt_b200 import plan as _plan
    T, R = len(dg.types), len(dg.edge_dict)
    _assert_bitwise(a, b)
    pa, pb = (_plan.get_plan(x[1], x[3], x[4], x[2], T, R) for x in (a, b))
    assert pa.type_count == pb.type_count and pa.pairs == pb.pairs and pa.n_edges == pb.n_edges


def _compare(dg, call, monkeypatch):
    """call(dg, generator) on the dense and the hashed state from the same generator state; returns the hashed batch."""
    dense = _as("dense", lambda: call(dg, _gen(7)), monkeypatch)
    assert dg.sampler_state["layout"] == "dense"
    hashed = _as("hashed", lambda: call(dg, _gen(7)), monkeypatch)
    assert dg.sampler_state["layout"] == "hashed" and dg.sampler_state["load"] <= 0.5
    assert len(dense) == len(hashed)
    for a, b in zip(dense, hashed):
        _assert_same(a, b, dg)
    return hashed


@pytest.mark.parametrize("features", [True, False])
@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("timed", [True, False])
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
def test_hashed_state_gives_the_dense_batch(name, B, timed, placement, features, monkeypatch):
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair(name, features)
    dg = dd if placement == "device" else dh
    inps = _inps(fx, fg, big, B, seed=B)
    tr = fx["time_range"] if timed else None
    _compare(dg, lambda g, gen: sampler.sample_subgraphs_cuda(g, tr, 4, 32, inps, gen), monkeypatch)


@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("rule", ["paper_field", "paper_venue", "author_disambiguation", "both_sides"])
def test_hashed_state_with_the_edge_masks(rule, placement, monkeypatch):
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair("sampler_large", True)
    dg = dd if placement == "device" else dh
    inps = _inps(fx, fg, big, 8, seed=3)
    mask = _rules(16)[rule]
    _compare(dg, lambda g, gen: sampler.sample_subgraphs_cuda(g, fx["time_range"], 3, 16, inps, gen, edge_mask=mask),
             monkeypatch)


@pytest.mark.parametrize("placement", ["device", "host"])
def test_hub_target_far_above_the_width(placement, monkeypatch):
    from pyhgt_b200 import sampler
    deg = 5000
    adj = {0: list(range(deg)), 1: list(range(0, deg, 7)), 2: [3, 5, 4999]}
    fg = sampler.FrozenGraph(_small(adj))
    tabs = {"paper": torch.randn(3, 12), "author": torch.randn(deg, 12)}
    dg = sampler.DeviceGraph(fg, _dev(), tabs, placement=placement)
    inps = [{"paper": np.array([[0, 2000], [1, 2000], [2, 2000]])}, {"paper": np.array([[0, 2000]])},
            {"author": np.array([[17, 2000], [4000, 2000]])}]
    out = _compare(dg, lambda g, gen: sampler.sample_subgraphs_cuda(g, {2000: True}, 3, 16, inps, gen), monkeypatch)
    assert out[0][7]["author"].numel() > 16


def test_an_overflowing_room_restarts_and_grows(monkeypatch):
    from pyhgt_b200 import sampler
    fx, fg, dd, _, big = _pair("sampler_large", True)
    inps = _inps(fx, fg, big, 8, seed=1)
    call = lambda g, gen: sampler.sample_subgraphs_cuda(g, fx["time_range"], 5, 64, inps, gen)
    dense = _as("dense", lambda: call(dd, _gen(2)), monkeypatch)
    dd.state_room = 0.01
    hashed = _as("hashed", lambda: call(dd, _gen(2)), monkeypatch)
    assert dd.sampler_state["restarts"] >= 1 and dd.state_room > 0.01
    for a, b in zip(dense, hashed):
        _assert_same(a, b, dd)
    room = dd.state_room
    again = _as("hashed", lambda: call(dd, _gen(2)), monkeypatch)
    assert dd.sampler_state["restarts"] == 0 and dd.state_room == room
    for a, b in zip(dense, again):
        _assert_same(a, b, dd)


def test_a_seed_past_the_dense_sort_limit(monkeypatch):
    """One isolated paper seed with id 2^31 + 5 in every member: the dense state would sort 8 x 2^31 ids per paper step.
    The rule picks the hashed state, and the batch is the dense one with that seed renamed to the first id past the
    graph, except for that seed's indxs entry."""
    from pyhgt_b200 import sampler
    fx, fg, dd, _, _ = _pair("sampler_large", False)
    huge, free = 2 ** 31 + 5, fg.n_ids["paper"]
    rng = np.random.RandomState(0)
    inps = []
    for b in range(8):
        ids = rng.choice(fg.n_ids["paper"], 12, replace=False)
        inps.append({"paper": np.stack([np.append(ids, huge), rng.randint(2000, 2016, 13)], 1)})
    renamed = []
    for inp in inps:
        p = inp["paper"].copy()
        p[12, 0] = free
        renamed.append({"paper": p})
    got = sampler.sample_subgraphs_cuda(dd, fx["time_range"], 4, 32, inps, _gen(4))
    assert dd.sampler_state["layout"] == "hashed"
    ref = _as("dense", lambda: sampler.sample_subgraphs_cuda(dd, fx["time_range"], 4, 32, renamed, _gen(4)),
              monkeypatch)
    for a, b in zip(got, ref):
        ia, ib = a[7]["paper"].clone(), b[7]["paper"].clone()
        assert int(ia[12]) == huge and int(ib[12]) == free
        ia[12] = free
        assert torch.equal(ia, ib)
        a[7]["paper"] = ib
        _assert_same(a, b, dd)
    with pytest.raises(ValueError, match="2\\^40"):
        sampler.sample_subgraphs_cuda(dd, fx["time_range"], 2, 8, [{"paper": np.array([[2 ** 40, 2010]])}], _gen(0))
