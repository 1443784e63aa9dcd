"""DeviceGraph(..., placement="host"): the CSR blocks and feature tables stay in page-locked host memory and the sampler
kernels read them in place.

  * every sampler entry point gives bitwise the batch of a device-placed graph from the same generator state, with and
    without features, time filter and the OAG scripts' edge masks, and the same cached plan per member;
  * a hub target (degree far above the width) goes through the single-read rebuild, and a rebuild whose hit records do
    not fit the scratch falls back to re-reading the lists with the same result;
  * building a host-placed graph puts only the per-block descriptors and per-type tables on the device, and leaves one
    host copy of each array: the FrozenGraph's blocks are the pinned copies, and the host sampler still works on them;
  * feature rows are gathered at any width: unaligned (OAG's 1169) and aligned rows of many 16-byte chunks;
  * a bad placement raises before any CUDA work."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import load_golden                    # noqa: E402
from tests.test_gpu_sampler import _dev, _gen, _small, _tables   # noqa: E402
from tests.test_gpu_sampler_batched import _assert_bitwise, _inps   # noqa: E402
from tests.test_gpu_sampler_mask import _rules           # noqa: E402
from tests.test_sampler import _GraphStub, _extractor    # noqa: E402


def _pair(name, features, width=8):
    """The fixture graph (plus a type without edges) placed on the device and in host memory, with the same tables."""
    from pyhgt_b200 import sampler
    fx = load_golden(name)
    g = _GraphStub(fx)
    g._t = g._t + ["never_seen_type"]
    fg = sampler.FrozenGraph(g)
    big = max(fg.n_ids.values()) + 7
    tabs = None
    if features:
        tabs = _tables(fg, g.get_types(), width=width)
        tabs["paper"] = torch.randn(big + 1, width)
        tabs["never_seen_type"] = torch.randn(4, width)
    return (fx, fg, sampler.DeviceGraph(fg, _dev(), tabs), sampler.DeviceGraph(fg, _dev(), tabs, placement="host"),
            big)


def _assert_same_batch(a, b, T, R):
    from pyhgt_b200 import plan as _plan
    _assert_bitwise(a, b)
    pa, pb = (_plan.get_plan(x[1], x[3], x[4], x[2], T, R) for x in (a, b))
    assert pa.type_count == pb.type_count and pa.pairs == pb.pairs and pa.n_edges == pb.n_edges


def _both(dd, dh, fn):
    """fn(graph, generator) on the device- and the host-placed graph from the same generator state."""
    return fn(dd, _gen(5)), fn(dh, _gen(5))


def _assert_records_fitted(dh):
    """The host graph's hit room grows only after a rebuild whose hit records overflowed, so an unchanged room means every
    write pass so far laid the edges out from the records (k_rb_write_hits), not by re-reading the lists."""
    from pyhgt_b200 import sampler
    assert dh.hit_room == sampler._HIT_ROOM


@pytest.mark.parametrize("features", [True, False])
@pytest.mark.parametrize("timed", [True, False])
def test_single_subgraph_equals_device_placement(features, timed):
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair("sampler_large", features)
    T, R = len(dd.types), len(dd.edge_dict)
    tr = fx["time_range"] if timed else None
    for inp in _inps(fx, fg, big, 5, seed=2):
        a, b = _both(dd, dh, lambda dg, g: sampler.sample_subgraph_cuda(dg, tr, 4, 32, inp, g))
        assert (b[0] is not None) == features
        _assert_same_batch(a, b, T, R)
    _assert_records_fitted(dh)


@pytest.mark.parametrize("features", [True, False])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_batch_equals_device_placement(B, features):
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair("sampler_large", features)
    T, R = len(dd.types), len(dd.edge_dict)
    inps = _inps(fx, fg, big, B)
    for tr in (fx["time_range"], None):
        a, b = _both(dd, dh, lambda dg, g: sampler.sample_subgraphs_cuda(dg, tr, 5, 64, inps, g))
        assert len(a) == len(b) == B
        for x, y in zip(a, b):
            _assert_same_batch(x, y, T, R)
    _assert_records_fitted(dh)


@pytest.mark.parametrize("rule", ["paper_field", "paper_venue", "author_disambiguation"])
def test_edge_masks_equal_device_placement(rule):
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair("sampler_large", True)
    T, R = len(dd.types), len(dd.edge_dict)
    inp = fx["inp"]
    mask = _rules(len(inp["paper"]))[rule]
    a, b = _both(dd, dh, lambda dg, g: sampler.sample_subgraph_cuda(dg, fx["time_range"], 4, 32, inp, g,
                                                                    edge_mask=mask))
    _assert_same_batch(a, b, T, R)
    for B in (3, 8):
        inps = _inps(fx, fg, big, B, seed=B)
        a, b = _both(dd, dh, lambda dg, g: sampler.sample_subgraphs_cuda(dg, None, 3, 16, inps, g, edge_mask=mask))
        for x, y in zip(a, b):
            _assert_same_batch(x, y, T, R)
    _assert_records_fitted(dh)


@pytest.mark.parametrize("width", [1169, 1028])
def test_feature_gather_at_wide_and_unaligned_widths(width):
    """1169 floats (OAG: 400 + 768 + 1) is not a multiple of 4, so rows take the 4-byte path; 1028 takes the 16-byte path
    with 257 chunks per row: three rounds of the 128-chunk loop and a partial last one."""
    from pyhgt_b200 import sampler
    fx, fg, dd, dh, big = _pair("sampler_large", True, width)
    T, R = len(dd.types), len(dd.edge_dict)
    inps = _inps(fx, fg, big, 3, seed=width)
    a, b = _both(dd, dh, lambda dg, g: sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 32, inps, g))
    for x, y in zip(a, b):
        assert x[0].shape[1] == width
        _assert_same_batch(x, y, T, R)


def test_hub_target_and_a_hit_scratch_that_does_not_fit():
    """Paper 0 has 5000 authors (width 16): its list spans many of the count pass's 256-neighbour rounds.  With no room
    reserved the hit records do not fit, the write pass re-reads the lists, the batch is the same, and the room grows so
    that the next batch fits."""
    from pyhgt_b200 import sampler
    deg = 5000
    adj = {0: list(range(deg)), 1: list(range(0, deg, 7)), 2: [3, 5, 4999]}
    g = _small(adj)
    fg = sampler.FrozenGraph(g)
    tabs = {"paper": torch.randn(3, 12), "author": torch.randn(deg, 12)}
    dd = sampler.DeviceGraph(fg, _dev(), tabs)
    dh = sampler.DeviceGraph(fg, _dev(), tabs, placement="host")
    T, R = len(dd.types), len(dd.edge_dict)
    inp = {"paper": np.array([[0, 2000], [1, 2000], [2, 2000]])}
    call = lambda dg, gen: sampler.sample_subgraphs_cuda(dg, {2000: True}, 3, 16, [inp] * 3, gen)
    dh.hit_room = 0.0
    a, b = _both(dd, dh, call)
    assert dh.hit_room > 0
    for x, y in zip(a, b):
        _assert_same_batch(x, y, T, R)
    room = dh.hit_room
    a, b = _both(dd, dh, call)
    assert dh.hit_room == room                            # this time the records fit
    for x, y in zip(a, b):
        _assert_same_batch(x, y, T, R)


def test_host_placement_puts_only_descriptors_on_the_device():
    from pyhgt_b200 import sampler
    fx = load_golden("sampler_large")
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types(), width=64)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    dh = sampler.DeviceGraph(fg, _dev(), tabs, placement="host")
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    NB, T = dh.n_blocks, len(dh.types)
    r512 = lambda n: 512 * math.ceil(n / 512)
    bound = r512(56 * NB) + r512(8 * T) + r512(8 * T) + r512(8 * T)   # blocks_dev, type ranges, feat_ptrs, feat_rows
    assert grown <= bound, (grown, bound)
    graph_bytes = sum(8 * (b.row_of.size + b.ptr.size + b.nbr.size + b.time.size)
                      for tes in fg.blocks.values() for rels in tes.values() for b in rels.values())
    graph_bytes += sum(4 * v.numel() for v in tabs.values())
    assert 8 * bound < graph_bytes, (bound, graph_bytes)
    for v in dh.features.values():
        assert v.device.type == "cpu" and v.is_pinned()
    for tes in fg.blocks.values():                        # the FrozenGraph's arrays are the pinned copies themselves
        for rels in tes.values():
            for blk in rels.values():
                for arr in (blk.row_of, blk.ptr, blk.nbr, blk.time):
                    assert any(arr is k for k in dh._keep) and torch.from_numpy(arr).is_pinned()
                assert blk.nbr_addr == blk.nbr.ctypes.data and blk.time_addr == blk.time.ctypes.data
    dd = sampler.DeviceGraph(fg, _dev(), tabs)
    for t in tabs:
        assert torch.equal(dd.features[t].cpu(), dh.features[t])


def test_bad_placement_raises_before_any_cuda_work():
    from pyhgt_b200 import _lib, sampler
    fx = load_golden("sampler")
    fg = sampler.FrozenGraph(_GraphStub(fx))
    torch.cuda.synchronize()
    before, launches = torch.cuda.memory_allocated(), _lib.kernel_launches()
    for bad in ("pinned", "HOST", None, ""):
        with pytest.raises(ValueError):
            sampler.DeviceGraph(fg, _dev(), placement=bad)
    assert torch.cuda.memory_allocated() == before and _lib.kernel_launches() == launches


def test_host_sampler_still_works_on_the_rebound_graph():
    """Building a host-placed graph rebinds the FrozenGraph's blocks to pinned copies (after the host sampler has cached
    its native block tables): the host sampler gives the same batch as before, also after the DeviceGraph is gone."""
    import gc
    from pyhgt_b200 import sampler
    fx = load_golden("sampler_large")
    fg = sampler.FrozenGraph(_GraphStub(fx))

    def host_batch():
        np.random.seed(3)
        return sampler.sample_subgraph(fg, fx["time_range"], 3, 16, fx["inp"], _extractor)

    before = host_batch()
    dh = sampler.DeviceGraph(fg, _dev(), placement="host")
    sampler.sample_subgraph_cuda(dh, fx["time_range"], 3, 16, fx["inp"], _gen(0))
    for after in (host_batch(), None):
        if after is None:
            del dh
            gc.collect()
            after = host_batch()
        for k in before[3]:
            assert np.array_equal(before[3][k], after[3][k]), k
        for t in before[2]:
            for s in before[2][t]:
                for r in before[2][t][s]:
                    assert np.array_equal(np.asarray(before[2][t][s][r]), np.asarray(after[2][t][s][r])), (t, s, r)
