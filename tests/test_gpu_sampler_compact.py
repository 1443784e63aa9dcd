"""The device sampler on compact graphs: 32-bit adjacency blocks and bf16 feature tables.

  * the same graph built all-wide (int64 blocks), all-narrow (int32 blocks) and mixed gives bitwise the same batches
    from sample_subgraphs_cuda: device and host placement, dense and hashed state, B = 1 and 8, with and without an edge
    mask and the time filter, on a graph with a block of None times;
  * bf16 tables give the fp32 tables' batch in every tensor but node_feature, and node_feature is the bf16-rounded fp32
    one widened back, bitwise: widths 128 (16-byte rows), 1169 and 37 (rows at every alignment, element-wise ends),
    both placements, both state layouts;
  * graph_bytes: the narrow adjacency holds half the wide one's bytes, bf16 tables half the fp32 ones."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import load_golden                    # noqa: E402
from tests.test_gpu_sampler import _dev, _gen, _tables    # noqa: E402
from tests.test_gpu_sampler_batched import _assert_bitwise, _inps   # noqa: E402
from tests.test_gpu_sampler_mask import _rules            # noqa: E402
from tests.test_sampler import _GraphStub                 # noqa: E402
from tests.test_sampler_compact_cpu import three_builds, with_none_times   # noqa: E402

_BUILDS = {}


def _graphs(placement, monkeypatch):
    """(fx, {"wide" | "narrow" | "mixed": DeviceGraph}, big) of sampler_large with None times in one block, the same
    fp32 tables everywhere; built once per placement."""
    from pyhgt_b200 import sampler
    if placement not in _BUILDS:
        fx = with_none_times(load_golden("sampler_large"))
        g = _GraphStub(fx)
        g._t = g._t + ["never_seen_type"]
        fgs = three_builds(g, monkeypatch)
        big = max(fgs["wide"].n_ids.values()) + 7
        tabs = _tables(fgs["wide"], g.get_types())
        tabs["paper"] = torch.randn(big + 1, 8, generator=torch.Generator().manual_seed(1))
        tabs["never_seen_type"] = torch.randn(4, 8, generator=torch.Generator().manual_seed(2))
        _BUILDS[placement] = (fx, {k: sampler.DeviceGraph(fg, _dev(), tabs, placement=placement)
                                   for k, fg in fgs.items()}, big)
    return _BUILDS[placement]


def _call(dg, layout, fn, monkeypatch):
    from pyhgt_b200 import sampler
    with monkeypatch.context() as m:
        m.setattr(sampler, "_FORCE_LAYOUT", layout)
        out = fn(dg, _gen(9))
    assert dg.sampler_state["layout"] == layout
    return out


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("timed", [True, False])
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("layout", ["dense", "hashed"])
@pytest.mark.parametrize("placement", ["device", "host"])
def test_wide_narrow_and_mixed_blocks_give_the_same_batch(placement, layout, B, timed, masked, monkeypatch):
    from pyhgt_b200 import sampler
    fx, dgs, big = _graphs(placement, monkeypatch)
    inps = _inps(fx, dgs["wide"].fg, big, B, seed=B + 2 * timed)
    tr = fx["time_range"] if timed else None
    mask = _rules(16)["both_sides"] if masked else None
    fn = lambda g, gen: sampler.sample_subgraphs_cuda(g, tr, 4, 32, inps, gen, edge_mask=mask)
    ref = _call(dgs["wide"], layout, fn, monkeypatch)
    assert sum(int(o[3].shape[1]) for o in ref) > 0
    for k in ("narrow", "mixed"):
        got = _call(dgs[k], layout, fn, monkeypatch)
        assert len(got) == len(ref)
        for a, b in zip(ref, got):
            _assert_bitwise(a, b)


def test_the_none_time_blocks_are_sampled_from(monkeypatch):
    """The blocks holding None times are narrow and lie in the sample, so the comparisons above read INT32_MIN
    entries."""
    from pyhgt_b200 import sampler
    fx, dgs, big = _graphs("device", monkeypatch)
    fg = dgs["narrow"].fg
    none_blocks = [b for tes in fg.blocks.values() for rels in tes.values() for b in rels.values() if b.has_none]
    assert none_blocks and all(b.narrow and (b.time == np.iinfo(np.int32).min).any() for b in none_blocks)
    rels = {r for tes in fg.blocks.values() for rs in tes.values() for r, b in rs.items() if b.has_none}
    out = sampler.sample_subgraphs_cuda(dgs["narrow"], fx["time_range"], 4, 32, _inps(fx, fg, big, 8), _gen(9))
    for r in rels:
        assert any(int((o[4] == dgs["narrow"].edge_dict[r]).sum()) > 0 for o in out), r


@pytest.mark.parametrize("layout", ["dense", "hashed"])
@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("width", [128, 1169, 37])
def test_bf16_tables_give_the_rounded_fp32_features(width, placement, layout, monkeypatch):
    from pyhgt_b200 import sampler
    fx = load_golden("sampler_large")
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    tabs = _tables(fg, g.get_types(), width=width, seed=width)
    tabs["paper"][0, :3] = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -9, -0.0])   # ties to even, signed zero
    d32 = sampler.DeviceGraph(fg, _dev(), tabs, placement=placement)
    d16 = sampler.DeviceGraph(fg, _dev(), tabs, placement=placement, feature_dtype=torch.bfloat16)
    assert all(v.dtype == torch.bfloat16 for v in d16.features.values())
    if placement == "host":
        assert all(v.device.type == "cpu" and v.is_pinned() for v in d16.features.values())
    inps = _inps(fx, fg, 0, 5, seed=width)[:2] + [{"paper": np.array([[0, 2010], [1, 2011]])}]
    fn = lambda dg, gen: sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 16, inps, gen)
    a, b = _call(d32, layout, fn, monkeypatch), _call(d16, layout, fn, monkeypatch)
    for x, y in zip(a, b):
        assert y[0].dtype == torch.float32 and y[0].shape == x[0].shape
        assert torch.equal(y[0], x[0].to(torch.bfloat16).float())
        _assert_bitwise((None,) + x[1:], (None,) + y[1:])
    f0 = b[2][0][int(b[2][5]["paper"][0])]                # member 2's first row: paper 0
    assert f0[:3].tolist() == [1.0, 1.0 + 2.0 ** -7, 0.0] and str(f0[2].item()) == "-0.0"


@pytest.mark.parametrize("placement", ["device", "host"])
def test_graph_bytes_halve(placement, monkeypatch):
    from pyhgt_b200 import sampler
    fx = load_golden("sampler_large")
    g = _GraphStub(fx)
    fgs = three_builds(g, monkeypatch)
    tabs = _tables(fgs["wide"], g.get_types(), width=24)
    wide = sampler.DeviceGraph(fgs["wide"], _dev(), tabs, placement=placement).graph_bytes
    narrow = sampler.DeviceGraph(fgs["narrow"], _dev(), tabs, placement=placement,
                                 feature_dtype=torch.bfloat16).graph_bytes
    elems = sum(b.row_of.size + b.ptr.size + b.nbr.size + b.time.size
                for tes in fgs["wide"].blocks.values() for rels in tes.values() for b in rels.values())
    assert wide == {"adjacency": 8 * elems, "features": 4 * 24 * sum(v.shape[0] for v in tabs.values()),
                    "placement": placement}
    assert 2 * narrow["adjacency"] == wide["adjacency"] and 2 * narrow["features"] == wide["features"]
    assert narrow["placement"] == placement
