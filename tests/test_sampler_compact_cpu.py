"""The FrozenGraph's 32-bit block format, without a GPU:

  * the format rule: ordinary blocks are narrow (int32 arrays), a block with one time past int32, or with an entry count,
    row count or id past the bound, keeps int64 arrays; a None time reads back as _NO_TIME;
  * the host sampler's three code paths give bitwise the same (feature, times, edge_list, indxs, texts) and RNG end state
    from an all-wide, an all-narrow and a mixed build of the same graph, None times included;
  * DeviceGraph.graph_bytes counts 4 bytes per element of a narrow block and 8 of a wide one."""
import copy
import types

import numpy as np
import pytest
import torch

from pyhgt_b200 import sampler
from tests.conftest import load_golden
from tests.test_sampler import _GraphStub, _extractor, _norm

ALL_WIDE = -1                                             # no block fits a negative bound


def _blocks(fg):
    return [blk for tes in fg.blocks.values() for rels in tes.values() for blk in rels.values()]


def with_none_times(fx, every=3):
    """The fixture with every `every`-th time of its first non-'self' block set to None (data.py:125-126)."""
    fx = dict(fx)
    fx["edge_list"] = el = copy.deepcopy(fx["edge_list"])
    for t_t, d1 in el.items():
        for s_t, d2 in d1.items():
            for r, tesr in d2.items():
                if r != "self" and tesr:
                    k = 0
                    for adl in tesr.values():
                        for sid in adl:
                            if k % every == 0:
                                adl[sid] = None
                            k += 1
                    return fx
    raise AssertionError("no block to put None times in")


def build(g, bound, monkeypatch):
    """FrozenGraph(g) with _NARROW_MAX = bound (None: the default)."""
    if bound is None:
        return sampler.FrozenGraph(g)
    with monkeypatch.context() as m:
        m.setattr(sampler, "_NARROW_MAX", bound)
        return sampler.FrozenGraph(g)


def mixed(g, monkeypatch):
    """A FrozenGraph of g whose blocks alternate between the narrow and the wide format (the fixtures' times make every
    block need the same bound, so no single bound mixes them)."""
    fg, wide = build(g, None, monkeypatch), build(g, ALL_WIDE, monkeypatch)
    k = 0
    for t_t, tes in fg.blocks.items():
        for s_t, rels in tes.items():
            for r in rels:
                if k % 2:
                    rels[r] = wide.blocks[t_t][s_t][r]
                k += 1
    return fg


def three_builds(g, monkeypatch):
    """{"wide", "narrow", "mixed"}: FrozenGraphs of g in which every block is wide, every block narrow, or both occur."""
    fgs = {"wide": build(g, ALL_WIDE, monkeypatch), "narrow": build(g, None, monkeypatch), "mixed": mixed(g, monkeypatch)}
    kinds = {k: {b.narrow for b in _blocks(fg)} for k, fg in fgs.items()}
    assert kinds == {"wide": {False}, "narrow": {True}, "mixed": {False, True}}, kinds
    return fgs


# ---- the format rule -------------------------------------------------------------------------------------------------

def test_ordinary_blocks_are_narrow():
    fg = sampler.FrozenGraph(_GraphStub(load_golden("sampler_large")))
    for blk in _blocks(fg):
        assert blk.narrow
        for a in (blk.row_of, blk.ptr, blk.nbr, blk.time):
            assert a.dtype == np.int32


def test_a_time_past_int32_keeps_the_block_wide():
    narrow = sampler._Block({0: {1: 2010, 2: 2011}, 1: {2: 2012}}, 2)
    wide = sampler._Block({0: {1: 2010, 2: 2 ** 33}, 1: {2: 2012}}, 2)
    assert narrow.narrow and not wide.narrow
    assert wide.time.dtype == np.int64 and wide.nbr.dtype == np.int64 and wide.time[1] == 2 ** 33
    for t in (2 ** 31 - 1, -2 ** 31 + 1):                 # the ends of the narrow time range
        assert sampler._Block({0: {1: t}}, 1).narrow
    for t in (2 ** 31, -2 ** 31):                         # INT32_MIN stands for None
        assert not sampler._Block({0: {1: t}}, 1).narrow
    assert not sampler._Block({0: {2 ** 31: 5}}, 1).narrow        # a neighbour id past int32


def test_none_times_of_a_narrow_block_read_back_as_no_time():
    blk = sampler._Block({0: {1: None, 2: 2011, 3: None}, 1: {2: 2012}}, 2)
    assert blk.narrow and blk.has_none
    assert blk.time.tolist() == [np.iinfo(np.int32).min, 2011, np.iinfo(np.int32).min, 2012]
    nbr, tm = blk.span(0, 4)
    assert nbr.dtype == np.int64 and tm.dtype == np.int64
    assert nbr.tolist() == [1, 2, 3, 2] and tm.tolist() == [sampler._NO_TIME, 2011, sampler._NO_TIME, 2012]
    assert blk.span(1, 3)[1].tolist() == [2011, sampler._NO_TIME]


def test_row_and_entry_counts_at_the_bound(monkeypatch):
    monkeypatch.setattr(sampler, "_NARROW_MAX", 4)
    assert sampler._Block({0: {1: 2, 2: 3, 3: 4, 4: 1}}, 1).narrow                  # 4 entries
    assert not sampler._Block({0: {1: 2, 2: 3, 3: 4, 4: 1}, 1: {1: 1}}, 2).narrow   # 5 entries
    assert sampler._Block({0: {0: 1}, 1: {0: 1}, 2: {0: 1}, 4: {0: 1}}, 5).narrow   # 4 rows, target id 4
    assert not sampler._Block({0: {0: 1}, 1: {0: 1}, 2: {0: 1}, 5: {0: 1}}, 6).narrow   # target id 5
    assert not sampler._Block({0: {0: 1}, 1: {0: 1}, 2: {0: 1}, 3: {0: 1}, 4: {0: 1}}, 5).narrow   # 5 rows
    assert not sampler._Block({0: {5: 1}}, 1).narrow                                  # neighbour id 5
    assert sampler._Block({0: {0: -4}}, 1).narrow and not sampler._Block({0: {0: -5}}, 1).narrow   # times
    blk = sampler._Block({0: {1: 2, 2: 3}, 3: {1: None}}, 4)
    assert blk.narrow and blk.row_of.tolist() == [0, -1, -1, 1] and blk.ptr.tolist() == [0, 2, 3]


# ---- the host sampler on every build -----------------------------------------------------------------------------------

@pytest.fixture(params=["batched", "slices", "numpy"])
def impl(request, monkeypatch):
    if request.param != "batched":
        monkeypatch.setattr(sampler, "_NATIVE_BATCH", [None, True])
    if request.param == "numpy":
        monkeypatch.setattr(sampler, "_NATIVE", [None, True])
    if request.param == "batched" and sampler._native_batch() is None:
        pytest.skip("libhgt_b200.so not built")
    return request.param


def _sample(fg, fx, depth, width, seed):
    np.random.seed(seed)
    out = sampler.sample_subgraph(fg, fx["time_range"], depth, width, fx["inp"], _extractor)
    return out, np.random.get_state()[1].copy()


def _assert_same_sample(a, b):
    (fa, ta, ea, ia, xa), rng_a = a
    (fb, tb, eb, ib, xb), rng_b = b
    assert np.array_equal(rng_a, rng_b)
    assert list(fa) == list(fb) and list(ia) == list(ib) and list(ta) == list(tb) and xa == xb
    for k in fa:
        for x, y in ((fa[k], fb[k]), (ta[k], tb[k]), (ia[k], ib[k])):
            assert x.dtype == y.dtype and np.array_equal(x, y), k
    na, nb = _norm(ea), _norm(eb)
    assert [x[:3] for x in na] == [x[:3] for x in nb]
    for x, y in zip(na, nb):
        assert np.asarray(x[3]).dtype == np.asarray(y[3]).dtype and np.array_equal(x[3], y[3]), x[:3]


@pytest.mark.parametrize("none_times", [False, True])
@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
def test_host_sampler_is_bitwise_the_same_on_every_build(name, none_times, impl, monkeypatch):
    fx = load_golden(name)
    if none_times:
        fx = with_none_times(fx)
    g = _GraphStub(fx)
    fgs = three_builds(g, monkeypatch)
    for depth, width, seed in ((2, 8, 3), (4, 32, 11)):
        ref = _sample(fgs["wide"], fx, depth, width, seed)
        for k in ("narrow", "mixed"):
            _assert_same_sample(ref, _sample(fgs[k], fx, depth, width, seed))


def test_edge_list_dtypes_are_those_of_the_wide_build(monkeypatch):
    """to_torch's inputs keep their dtypes: the sampled edge blocks are int64 [E, 2] arrays on the narrow build too."""
    fx = load_golden("sampler")
    fgs = three_builds(_GraphStub(fx), monkeypatch)
    (_, _, el, _, _), _ = _sample(fgs["narrow"], fx, 2, 8, 0)
    for t in el:
        for s in el[t]:
            for r in el[t][s]:
                assert np.asarray(el[t][s][r]).dtype == np.int64


# ---- graph_bytes -------------------------------------------------------------------------------------------------------

def _bytes_of(fg, features, placement):
    """DeviceGraph.graph_bytes of a graph holding fg's block arrays and the given tables (no device needed)."""
    held = types.SimpleNamespace(_adjacency=[a for b in _blocks(fg) for a in (b.row_of, b.ptr, b.nbr, b.time)],
                                 features=features, placement=placement)
    return sampler.DeviceGraph.graph_bytes.fget(held)


def test_graph_bytes_counts_four_bytes_per_narrow_element(monkeypatch):
    fx = load_golden("sampler_large")
    fgs = three_builds(_GraphStub(fx), monkeypatch)
    elems = sum(b.row_of.size + b.ptr.size + b.nbr.size + b.time.size for b in _blocks(fgs["wide"]))
    tabs = {"paper": torch.zeros(10, 6), "author": torch.zeros(3, 6)}
    wide = _bytes_of(fgs["wide"], tabs, "host")
    narrow = _bytes_of(fgs["narrow"], {t: v.to(torch.bfloat16) for t, v in tabs.items()}, "host")
    assert wide == {"adjacency": 8 * elems, "features": 4 * 13 * 6, "placement": "host"}
    assert narrow == {"adjacency": 4 * elems, "features": 2 * 13 * 6, "placement": "host"}
    mixed = _bytes_of(fgs["mixed"], None, "device")
    assert 4 * elems < mixed["adjacency"] < 8 * elems and mixed["features"] == 0
    assert mixed["adjacency"] == sum((4 if b.narrow else 8) * (b.row_of.size + b.ptr.size + b.nbr.size + b.time.size)
                                     for b in _blocks(fgs["mixed"]))


def test_bad_feature_dtype_raises_before_any_cuda_work():
    fg = sampler.FrozenGraph(_GraphStub(load_golden("sampler")))
    with pytest.raises(ValueError, match="feature_dtype"):
        sampler.DeviceGraph(fg, "cuda:0", feature_dtype=torch.float16)
