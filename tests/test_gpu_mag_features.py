"""sampler.mag_features (csrc/features.cu) against the ogbn-mag preprocessing script and a float64 restatement.

* tests/golden/mag_features*.pt (oracle/make_mag_features_golden.py) holds graph.node_feature as the unmodified script
  computes it on two small OGB-style edge sets: a pair repeated inside a key, a pair under two relations between the
  same types, an author with no paper, nodes without edges (num_nodes above the largest id), a type the script makes
  no table for, F = 128 and F = 37, and years past 2^31 that make some blocks wide.  Each is rebuilt with from_edges on
  both placements, with the default widths and with every block wide, and mag_features must give the script's values
  rounded to float32 within 1 ulp, with -inf and zero entries exact, bitwise the same on a second call.
* The ogbn-mag-sized synthetic graph against float64 index_add_ sums over the graph's own blocks.
* set_features of those tables samples bitwise the batches of from_edges(..., features=the same tables), fp32 and bf16.

Single-rule faults this file catches (each run once against the suite, every one failing): counting a pair that two
relations share once, averaging the paper table with its degree column, leaving rev_ blocks out of deg, dividing the
sums by deg instead of the pair count."""
import numpy as np
import pytest
import torch

from tests.conftest import load_golden
from tests.test_gpu_graph_ingest import assert_same_batches, mag_shaped_edges

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def ogb_edges(case):
    """The fixture's keys as from_edges items, with the times the script gives them: the paper end's year, None for
    keys without a paper end."""
    years = case["years"]
    out = []
    for (s_t, r, t_t), ei in case["edges"]:
        tm = years[ei[0]] if s_t == "paper" else years[ei[1]] if t_t == "paper" else None
        out.append(((s_t, r, t_t), ei, tm))
    return out


def _ordered(a):
    """float32 bits as integers whose order is the values' order (for ulp distances)."""
    b = a.contiguous().view(torch.int32).to(torch.int64)
    return torch.where(b < 0, -(b & 0x7FFFFFFF), b)


def assert_within_1ulp(got, ref64, what):
    """got (float32) within 1 ulp of ref64 rounded to float32; -inf and zeros of the reference exactly equal."""
    ref = ref64.to(torch.float32)
    assert got.dtype == torch.float32 and got.shape == ref.shape, (what, got.dtype, got.shape, ref.shape)
    exact = torch.isinf(ref) | (ref == 0)
    assert torch.equal(got[exact], ref[exact]), what
    assert torch.isfinite(got[~exact]).all(), what
    d = (_ordered(got) - _ordered(ref)).abs()[~exact]
    assert d.numel() == 0 or int(d.max()) <= 1, (what, int(d.max()))


def check_against_script(case, dg, x):
    from pyhgt_b200 import sampler
    ref = case["node_feature"]
    got = sampler.mag_features(dg, x, case["num_nodes"])
    assert list(got) == list(ref)
    for t in ref:
        assert got[t].device == dg.device
        assert_within_1ulp(got[t].cpu(), ref[t], t)
    assert torch.equal(got["paper"][:, :-1].cpu(), case["x_paper"])
    again = sampler.mag_features(dg, x, case["num_nodes"])
    assert all(torch.equal(got[t], again[t]) for t in ref)
    return got


@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("widths", ["default", "wide"])
@pytest.mark.parametrize("name", ["small", "mixed"])
def test_matches_the_preprocessing_script(name, widths, placement, monkeypatch):
    from pyhgt_b200 import sampler
    if widths == "wide":
        monkeypatch.setattr(sampler, "_NARROW_MAX", -1)
    case = load_golden("mag_features")[name]
    dg = sampler.DeviceGraph.from_edges(ogb_edges(case), list(case["num_nodes"]), _dev(), placement=placement)
    narrow = [bool(c.skip & 2) for c in dg._cblocks]
    if widths == "wide":
        assert not any(narrow)
    elif name == "mixed":
        assert any(narrow) and not all(narrow)
    else:
        assert all(narrow)
    x = case["x_paper"]
    check_against_script(case, dg, x if placement == "host" else x.to(_dev()))
    if name == "mixed":
        assert "venue" not in sampler.mag_features(dg, x, case["num_nodes"])


def _pairs(dg, t, s=None):
    """(target ids, source ids) of every entry of dg's blocks into t (from s), block by block, on the device."""
    dev = dg.device
    out = []
    for b, (ti, si, _) in enumerate(dg.blocks):
        if dg.types[ti] != t or (s is not None and dg.types[si] != s):
            continue
        row_of, ptr, nbr = (torch.as_tensor(a).to(dev, torch.int64) for a in dg._adjacency[4 * b:4 * b + 3])
        ids = torch.nonzero(row_of >= 0).squeeze(1)
        rows = row_of[ids]
        lens = ptr[rows + 1] - ptr[rows]
        tgt = torch.repeat_interleave(ids, lens)
        first = torch.repeat_interleave(ptr[rows], lens)
        before = torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)
        out.append((tgt, nbr[first + torch.arange(tgt.numel(), device=dev) - before]))
    return out


def restate(dg, x64, num_nodes):
    """The script's rules in float64 over dg's blocks: {type: [num_nodes, F + 1] float64}."""
    dev = dg.device
    F = x64.shape[1]

    def deg(t):
        d = torch.zeros(num_nodes[t], dtype=torch.int64, device=dev)
        for tgt, _ in _pairs(dg, t):
            d += torch.bincount(tgt, minlength=num_nodes[t])
        return torch.log10(d.to(torch.float64)).unsqueeze(1)

    def mean(t, s, src):
        acc = torch.zeros(num_nodes[t], F, dtype=torch.float64, device=dev)
        cnt = torch.zeros(num_nodes[t], dtype=torch.float64, device=dev)
        for tgt, nb in _pairs(dg, t, s):
            for c in range(0, tgt.numel(), 1 << 20):
                acc.index_add_(0, tgt[c:c + (1 << 20)], src[nb[c:c + (1 << 20)]])
            cnt.index_add_(0, tgt, torch.ones_like(tgt, dtype=torch.float64))
        return acc / cnt.clamp(min=1).unsqueeze(1)

    out = {"paper": torch.cat([x64, deg("paper")], 1)}
    means = {}
    for t in num_nodes:
        if t not in ("paper", "institution"):
            means[t] = mean(t, "paper", x64)
            out[t] = torch.cat([means[t], deg(t)], 1)
    out["institution"] = torch.cat([mean("institution", "author", means["author"]), deg("institution")], 1)
    return out


def test_ogbn_mag_sized_against_float64():
    """synth.make_mag_shaped(1.0) (21.1 M edges, 42.2 M with rev_), OGB's num_nodes, F = 128.  The float64 sums of the
    restatement run in another order, so an entry may differ by one float32 ulp, plus 1e-13 where a mean nearly
    cancels to zero."""
    from pyhgt_b200 import sampler, synth
    edges, types = mag_shaped_edges()
    num_nodes = dict(zip(types, synth.MAG_NODE_COUNTS))
    dev = _dev()
    dg = sampler.DeviceGraph.from_edges(edges, types, dev)
    x = torch.randn(num_nodes["paper"], 128, generator=torch.Generator().manual_seed(5)).to(dev)
    got = sampler.mag_features(dg, x, num_nodes)
    ref = restate(dg, x.double(), num_nodes)
    assert list(got) == ["paper", "author", "field", "institution"] == list(ref)
    for t in ref:
        r32 = ref[t].to(torch.float32)
        assert got[t].shape == r32.shape
        inf = torch.isinf(r32)
        assert torch.equal(got[t][inf], r32[inf]) and inf[:, :-1].sum() == 0, t
        ulp = torch.abs(torch.nextafter(r32, torch.full_like(r32, float("inf"))) - r32)
        err = (got[t].double() - ref[t]).abs()[~inf]
        assert bool((err <= ulp[~inf].double() + 1e-13).all()), (t, float(err.max()))
        zero_rows = (ref[t][:, :-1] == 0).all(1)
        assert bool((got[t][zero_rows, :-1] == 0).all()), t


@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("feature_dtype", [None, torch.bfloat16])
def test_set_features_samples_as_features_given_to_the_constructor(feature_dtype, placement):
    from pyhgt_b200 import sampler
    case = load_golden("mag_features")["small"]
    edges, types = ogb_edges(case), list(case["num_nodes"])
    probe = sampler.DeviceGraph.from_edges(edges, types, _dev())
    tabs = sampler.mag_features(probe, case["x_paper"], case["num_nodes"])
    ref = sampler.DeviceGraph.from_edges(edges, types, _dev(), features=tabs, placement=placement,
                                         feature_dtype=feature_dtype)
    got = sampler.DeviceGraph.from_edges(edges, types, _dev(), placement=placement, feature_dtype=feature_dtype)
    assert got.features is None
    got.set_features(sampler.mag_features(got, case["x_paper"], case["num_nodes"]))
    assert got.feat_dim == ref.feat_dim == 129 and list(got.features) == list(ref.features)
    for t in ref.features:
        assert got.features[t].dtype == ref.features[t].dtype
        assert torch.equal(got.features[t].cpu(), ref.features[t].cpu())
    assert torch.equal(got.feat_rows, ref.feat_rows) and torch.equal(got.feat_ptrs != 0, ref.feat_ptrs != 0)
    years = {y: True for y in range(2000, 2020)}
    assert_same_batches(got, ref, "paper", years, feature_dtype=feature_dtype)
    assert_same_batches(got, ref, "author", years, feature_dtype=feature_dtype)


def test_refusals_on_a_built_graph():
    from pyhgt_b200 import sampler
    case = load_golden("mag_features")["small"]
    edges, types, nn = ogb_edges(case), list(case["num_nodes"]), case["num_nodes"]
    dg = sampler.DeviceGraph.from_edges(edges, types, _dev())
    bad = {"paper": torch.zeros(3, 4), "author": torch.zeros(3, 5)}
    with pytest.raises(ValueError, match="same width") as a:
        dg.set_features(bad)
    with pytest.raises(ValueError, match="same width") as b:
        sampler.DeviceGraph.from_edges(edges, types, _dev(), features=bad)
    assert str(a.value) == str(b.value)
    for t in types:
        if t != "paper":
            with pytest.raises(ValueError, match="below the graph's id range of %r" % t):
                sampler.mag_features(dg, case["x_paper"], {**nn, t: dg.n_ids[dg.slot[t]] - 1})
    with pytest.raises(ValueError, match="x_paper"):
        sampler.mag_features(dg, case["x_paper"][:-1], nn)
    with pytest.raises(ValueError, match="below"):
        sampler.mag_features(dg, case["x_paper"][:-7], {**nn, "paper": nn["paper"] - 7})
    with pytest.raises(ValueError, match="x_paper"):
        sampler.mag_features(dg, case["x_paper"].half(), nn)
