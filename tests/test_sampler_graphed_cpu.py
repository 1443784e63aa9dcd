"""sampler.GraphedSampler and graph_signature_for without a GPU: argument checks, bound arithmetic, the C symbols."""
import ctypes as _c

import numpy as np
import pytest


def test_the_fixed_shape_entry_points_are_bound_and_check_their_arguments():
    from pyhgt_b200 import _lib
    _lib.load()
    for name, n in (("hgt_gsample_layer_order", 9), ("hgt_gsample_graphed_layout", 21),
                    ("hgt_gsample_graphed_rows", 5), ("hgt_gsample_graphed_pad", 11)):
        assert len(_lib.SIGNATURES[name]) == n, name
        with pytest.raises(_lib.HgtError, match=name):        # NULL tables
            _lib.call(name, *[None if t is _c.c_void_p else 1 for t in _lib.SIGNATURES[name]])


def test_hash_select_refuses_more_positions_than_members_times_room():
    """n_total may exceed sel_off[B] (padding) but not B x max_room: one position more is refused as a bad argument,
    exactly B x max_room gets past the argument check (to the workspace check: no workspace is given)."""
    from pyhgt_b200 import _lib, sampler
    st = sampler._GHashState(2, 3, *([8] * 18))              # 3 members; non-NULL (never dereferenced) pointers
    args = lambda n_total: (_c.byref(st), 8, 8, 8, n_total, 10, 4, 8, 8, 8, 8, None, 0, None)
    with pytest.raises(_lib.HgtError, match="bad arguments"):
        _lib.call("hgt_gsample_hash_select", *args(31))
    with pytest.raises(_lib.HgtError, match="workspace too small"):
        _lib.call("hgt_gsample_hash_select", *args(30))


class _FakeDG:
    def __init__(self, placement="device", features=True):
        import torch
        self.placement = placement
        self.features = {"paper": None} if features else None
        self.feature_dtype = torch.float32
        self.types = ["paper", "author"]
        self.slot = {"paper": 0, "author": 1}
        self.edge_dict = {"AP_write": 0, "rev_AP_write": 1, "self": 2}
        self.blocks = [(0, 1, "AP_write"), (1, 0, "rev_AP_write")]
        self.n_blocks = 2
        self.feat_dim = 8
        self.n_ids = [1000, 50]
        self.state_room = 64.0
        self.device = "cpu"


def _sig(**kw):
    from pyhgt_b200 import graphed
    args = dict(type_counts=[300, 60], n_edges=900, pairs=[(0, 2), (1, 2), (1, 0), (0, 1)], num_relations=3,
                feat_dim=8)
    args.update(kw)
    return graphed.GraphSignature(**args)


def test_constructor_refusals():
    from pyhgt_b200 import sampler
    with pytest.raises(ValueError, match="placement='host'"):
        sampler.GraphedSampler(_FakeDG("host"), _sig(), 2, 16, {"paper": 8})
    with pytest.raises(ValueError, match="feature tables"):
        sampler.GraphedSampler(_FakeDG(features=False), _sig(), 2, 16, {"paper": 8})
    with pytest.raises(ValueError, match="the signature has"):
        sampler.GraphedSampler(_FakeDG(), _sig(feat_dim=4), 2, 16, {"paper": 8})
    with pytest.raises(KeyError, match="venue"):
        sampler.GraphedSampler(_FakeDG(), _sig(), 2, 16, {"venue": 8})
    with pytest.raises(ValueError, match="largest seed count"):
        sampler.GraphedSampler(_FakeDG(), _sig(), 2, 16, {"paper": 0})
    with pytest.raises(KeyError, match="edge_mask"):
        sampler.GraphedSampler(_FakeDG(), _sig(), 2, 16, {"paper": 8}, edge_mask={("paper", "venue", "x"): (1, 0)})


def test_bounds_follow_the_declared_seeds_depth_and_width():
    """The sizes the constructor fixes: layer capacity min(id range + seeds, seeds + depth x width), hashed rooms from
    state_room (at most twice the id range), the sort size B x the largest room, and the count slots."""
    from pyhgt_b200 import sampler
    dg = _FakeDG()
    bd = sampler._graphed_bounds(dg, [(0, 8)], 2, 16, 3)
    assert bd["layer_capacity"].tolist() == [40, 32]
    assert bd["region_entries"].tolist() == [min(2 * 1008, 64 * 56), min(2 * 50, 64 * 48)]
    assert bd["max_room"] == 2016 and bd["sort_positions"] == 3 * 2016
    assert bd["count_slots"] == 3 * (40 + 32)                # blocks: paper <- author, author <- paper
    dg.n_ids = [10, 50]
    assert sampler._graphed_bounds(dg, [(0, 8)], 2, 16, 1)["layer_capacity"].tolist() == [18, 32]
    dg.state_room = 1.0
    assert sampler._graphed_bounds(dg, [(0, 8)], 2, 16, 1)["region_entries"].tolist() == [34, 48]
    assert sampler._graphed_bounds(dg, [(0, 8)], 2, 16, 1, state_room=1e9)["region_entries"].tolist() == [36, 100]
    with pytest.raises(ValueError, match="int32 sort values"):
        sampler._graphed_bounds(_FakeDG(), [(0, 8)], 2, 16, 2 ** 21)


def test_seed_counts_over_the_declared_maximum_are_refused():
    """stage() checks seeds on the host before it touches any buffer."""
    from pyhgt_b200 import sampler
    gs = sampler.GraphedSampler.__new__(sampler.GraphedSampler)
    gs.dg, gs.B, gs.T, gs.decl = _FakeDG(), 1, 2, [(0, 4)]
    with pytest.raises(ValueError, match="more than the declared 4"):
        gs.stage({"paper": np.stack([np.arange(5), np.zeros(5, np.int64)], 1)})
    with pytest.raises(ValueError, match="was not declared"):
        gs.stage({"author": np.array([[1, 0]])})
    with pytest.raises(ValueError, match="2 seed dicts for 1 members"):
        gs.stage([{"paper": np.array([[1, 0]])}] * 2)


def test_pairs_of_a_graph_are_its_blocks_and_self():
    from pyhgt_b200 import sampler
    assert sampler._mag_pairs(_FakeDG()) == [(0, 1), (0, 2), (1, 0), (1, 2)]


def test_graph_signature_for_takes_the_largest_probe_times_members_and_slack(monkeypatch):
    """On a host-built graph (the fake one): the probes' per-type maximum and edge maximum, times members x (1 + slack),
    rounded up, and every block's pair plus 'self' on every type."""
    import torch
    from pyhgt_b200 import sampler
    probes = [(torch.tensor([0, 0, 0, 1]), 5), (torch.tensor([0, 1, 1]), 9)]
    seen = {}

    def fake(dg, time_range, depth, width, inps, generator=None, edge_mask=None, feature_dtype=None):
        seen["args"] = (time_range, depth, width, len(inps), edge_mask)
        return [(None, nt, None, None, torch.zeros(e, dtype=torch.int64)) for nt, e in probes]

    monkeypatch.setattr(sampler, "sample_subgraphs_cuda", fake)
    sig = sampler.graph_signature_for(_FakeDG(), 2, 16, [{}, {}], 0.5, members=2, time_range={2000: True})
    assert seen["args"] == ({2000: True}, 2, 16, 2, None)
    assert sig.type_counts == [9, 6] and sig.n_edges == 27
    assert sig.pairs == [(0, 1), (0, 2), (1, 0), (1, 2)] and sig.feat_dim == 8
    with pytest.raises(ValueError, match="probe"):
        sampler.graph_signature_for(_FakeDG(), 2, 16, [], 0.5)
