"""DeviceGraph.from_edges against the dict path it replaces.

The oracle replays the ogbn-mag preprocessing loop (preprocess_ogbn_mag.py:29-42) on the same arrays into a reference
dict graph, freezes it (FrozenGraph) and uploads it (DeviceGraph).  Every case asserts, bitwise, the block list,
edge_dict, n_ids, every block's row_of / ptr / nbr / time arrays with their dtypes and flags, and the feature tables;
then that sample_subgraphs_cuda gives bitwise the same batches from both graphs (B = 1 and 8, with an edge mask, and
with bf16 tables).  Cases: the MAG schema of scripts/gpu_sampler_bench.py at a small scale, duplicate pairs with
different times, None-time and 'self' blocks, an empty key, same-type relations, ids with gaps, all-wide and mixed
widths (a lowered _NARROW_MAX), reverse=False, both placements.  One more test builds the ogbn-mag-sized synthetic
graph (21.1 M edges, 42.2 M with rev_) and samples 32 subgraphs from it."""
from collections import defaultdict

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F = 16


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


class _Graph:
    """The parts of pyHGT's Graph the freezing and upload read: edge_list, get_types, get_meta_graph (data.py:63-73)."""

    def __init__(self, edge_list, types):
        self.edge_list, self._t = edge_list, list(types)

    def get_types(self):
        return self._t

    def get_meta_graph(self):
        return [(t, s, r) for t in self.edge_list for s in self.edge_list[t] for r in self.edge_list[t][s]]


def dict_graph(edges, types, reverse=True):
    """The preprocessing loop: key by key, elist[t][s] = time then rlist[s][t] = time per edge, in array order."""
    el = defaultdict(lambda: defaultdict(lambda: defaultdict(lambda: defaultdict(dict))))
    for (s_t, r, t_t), ei, tm in edges:
        elist = el[t_t][s_t][r]
        rlist = el[s_t][t_t]["rev_" + r] if reverse else None
        src, dst = ei[0].tolist(), ei[1].tolist()
        times = tm.tolist() if tm is not None else [None] * len(src)
        for s_id, t_id, year in zip(src, dst, times):
            elist[t_id][s_id] = year
            if reverse:
                rlist[s_id][t_id] = year
    return _Graph(el, types)


def _np(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def assert_same_graph(got, ref):
    assert got.fg is None
    assert got.types == ref.types and got.blocks == ref.blocks and got.n_blocks == ref.n_blocks
    assert got.edge_dict == ref.edge_dict and list(got.edge_dict) == list(ref.edge_dict)
    assert got.n_ids == ref.n_ids
    assert got.max_type_blocks == ref.max_type_blocks
    assert torch.equal(got.type_block_range, ref.type_block_range)
    for a, b in zip(got._cblocks, ref._cblocks):
        assert (a.n_row_of, a.tgt_type, a.src_type, a.skip, a.rel) == (b.n_row_of, b.tgt_type, b.src_type, b.skip, b.rel)
    assert len(got._adjacency) == len(ref._adjacency) == 4 * ref.n_blocks
    for i, (a, b) in enumerate(zip(got._adjacency, ref._adjacency)):
        a, b = _np(a), _np(b)
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), (ref.blocks[i // 4], i % 4)
    assert got.graph_bytes == ref.graph_bytes
    assert (got.features is None) == (ref.features is None)
    if ref.features is not None:
        assert set(got.features) == set(ref.features) and got.feat_dim == ref.feat_dim
        for t in ref.features:
            assert torch.equal(got.features[t].cpu(), ref.features[t].cpu())
        assert torch.equal(got.feat_rows, ref.feat_rows)


def _assert_same_batch(a, b):
    for x, y in zip(a[:5], b[:5]):
        assert (x is None and y is None) or (x.dtype == y.dtype and torch.equal(x, y))
    assert a[5] == b[5] and a[6] == b[6]
    for k in (7, 8):
        assert list(a[k]) == list(b[k]) and all(torch.equal(a[k][t], b[k][t]) for t in a[k])


def _tables(n_ids, types, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {t: torch.randn(max(n, 1) + 3, F, generator=g) for t, n in zip(types, n_ids)}


def build_both(edges, types, placement="device", reverse=True, features=True, feature_dtype=None):
    """(from_edges graph, dict-path graph) with the same feature tables."""
    from pyhgt_b200 import sampler
    fg = sampler.FrozenGraph(dict_graph(edges, types, reverse))
    tabs = _tables([fg.n_ids.get(t, 0) for t in types], types) if features else None
    ref = sampler.DeviceGraph(fg, _dev(), tabs, placement=placement, feature_dtype=feature_dtype)
    got = sampler.DeviceGraph.from_edges(edges, types, _dev(), reverse=reverse, features=tabs, placement=placement,
                                         feature_dtype=feature_dtype)
    return got, ref


def assert_same_batches(got, ref, seed_type, time_range, mask=None, feature_dtype=None, seeds=None):
    from pyhgt_b200 import sampler
    n = ref.n_ids[ref.slot[seed_type]]
    rng = np.random.RandomState(n)
    inps = []
    for _ in range(8):
        ids = seeds if seeds is not None else rng.choice(n, min(n, 6), replace=False)
        tms = rng.randint(2000, 2016, len(ids))
        inps.append({seed_type: np.stack([ids, tms], 1)})
    edges = 0
    for B in (1, 8):
        for m in (None, mask) if mask else (None,):
            a = sampler.sample_subgraphs_cuda(ref, time_range, 3, 8, inps[:B], torch.Generator().manual_seed(B),
                                              edge_mask=m, feature_dtype=feature_dtype)
            b = sampler.sample_subgraphs_cuda(got, time_range, 3, 8, inps[:B], torch.Generator().manual_seed(B),
                                              edge_mask=m, feature_dtype=feature_dtype)
            assert len(a) == len(b) == B
            for x, y in zip(a, b):
                _assert_same_batch(x, y)
                edges += int(x[3].shape[1])
    assert edges > 0


def mag_edges(P=2000, A=1200, Fi=160, V=50, seed=0, times=True):
    """scripts/gpu_sampler_bench.py's MAG schema as typed arrays: heavy-tailed citations, authorship and fields."""
    rng = np.random.RandomState(seed)
    year = rng.randint(1990, 2021, P)

    def key(s_t, r, t_t, src, dst, tm):
        ei = torch.from_numpy(np.stack([src, dst]).astype(np.int64))
        return (s_t, r, t_t), ei, (torch.from_numpy(tm.astype(np.int64)) if times else None)

    cited = (rng.pareto(1.2, 4 * P) * 50).astype(np.int64) % P
    citing = rng.randint(0, P, 4 * P)
    pa = rng.randint(0, P, 3 * P)
    au = (rng.pareto(1.5, 3 * P) * 30).astype(np.int64) % A
    pf = rng.randint(0, P, 3 * P)
    fi = (rng.pareto(1.0, 3 * P) * 20).astype(np.int64) % Fi
    return [key("paper", "PP_cite", "paper", cited, citing, year[citing]),
            key("author", "AP_write", "paper", au, pa, year[pa]),
            key("field", "PF_in_L2", "paper", fi, pf, year[pf]),
            key("venue", "PV_Journal", "paper", rng.randint(0, V, P), np.arange(P), year)]


TYPES = ["paper", "author", "field", "venue"]
YEARS = {y: True for y in range(1990, 2016)}
MASK = {("paper", "field", "PF_in_L2"): (6, 0), ("field", "paper", "rev_PF_in_L2"): (0, 6)}


@pytest.mark.parametrize("placement", ["device", "host"])
def test_mag_schema(placement):
    got, ref = build_both(mag_edges(), TYPES, placement)
    assert_same_graph(got, ref)
    assert_same_batches(got, ref, "paper", YEARS, MASK)


@pytest.mark.parametrize("placement", ["device", "host"])
def test_bf16_tables(placement):
    got, ref = build_both(mag_edges(seed=1), TYPES, placement, feature_dtype=torch.bfloat16)
    assert_same_graph(got, ref)
    assert_same_batches(got, ref, "paper", YEARS, feature_dtype=torch.bfloat16)
    assert_same_batches(got, ref, "paper", YEARS)


def _dup_edges(seed, n_ids=40, n=3000, time_hi=10):
    """Pairs drawn from a small id range (most repeat), each with its own time."""
    g = torch.Generator().manual_seed(seed)
    ei = torch.randint(0, n_ids, (2, n), generator=g)
    return ei, torch.randint(2000, 2000 + time_hi, (n,), generator=g)


@pytest.mark.parametrize("placement", ["device", "host"])
def test_duplicate_pairs_keep_first_place_and_last_time(placement):
    e1, t1 = _dup_edges(1)
    e2, t2 = _dup_edges(2, n_ids=25)
    edges = [(("paper", "cites", "paper"), e1, t1), (("author", "writes", "paper"), e2, t2)]
    got, ref = build_both(edges, ["paper", "author"], placement)
    assert_same_graph(got, ref)
    blk = ref.fg.blocks["paper"]["paper"]["cites"]
    assert blk.ptr[-1] < e1.shape[1]                      # repeats were merged
    assert_same_batches(got, ref, "paper", {y: True for y in range(2000, 2006)})


@pytest.mark.parametrize("placement", ["device", "host"])
def test_none_times_self_blocks_empty_keys(placement):
    """None-time keys, a 'self' key (reverse=True also makes 'rev_self'), an empty key in the middle, a same-type
    relation, and a type that only occurs as a seed type's neighbour."""
    g = torch.Generator().manual_seed(3)
    P, A = 300, 120
    ids = torch.arange(P)
    edges = [(("paper", "self", "paper"), torch.stack([ids, ids]), None),
             (("author", "writes", "paper"), torch.stack([torch.randint(0, A, (900,), generator=g),
                                                        torch.randint(0, P, (900,), generator=g)]), None),
             (("venue", "empty", "paper"), torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64)),
             (("paper", "cites", "paper"), torch.randint(0, P, (2, 1500), generator=g),
              torch.randint(2000, 2016, (1500,), generator=g))]
    types = ["paper", "author", "venue", "unused"]
    got, ref = build_both(edges, types, placement)
    assert_same_graph(got, ref)
    assert [r for _, _, r in ref.blocks].count("self") == 1
    assert_same_batches(got, ref, "paper", YEARS)
    assert_same_batches(got, ref, "paper", None)


@pytest.mark.parametrize("placement", ["device", "host"])
def test_ids_with_gaps_and_reverse_false(placement):
    """Strided and offset ids (row_of spans the largest id; a source type's range reaches past its target ids), and
    keys without rev_ twins."""
    g = torch.Generator().manual_seed(4)
    src = torch.randint(0, 50, (800,), generator=g) * 997 + 13
    dst = torch.randint(0, 60, (800,), generator=g) * 131 + 5
    a_src = torch.randint(0, 40, (500,), generator=g) * 50_021
    edges = [(("paper", "cites", "paper"), torch.stack([src, dst]), torch.randint(2000, 2016, (800,), generator=g)),
             (("author", "writes", "paper"), torch.stack([a_src, dst[:500]]), None),
             (("paper", "written_by", "author"), torch.stack([dst[:300], a_src[:300]]),
              torch.randint(2000, 2016, (300,), generator=g))]
    for reverse in (True, False):
        got, ref = build_both(edges, ["paper", "author"], placement, reverse=reverse)
        assert_same_graph(got, ref)
        seeds = np.unique(dst[:40].numpy())[:6]
        assert_same_batches(got, ref, "paper", YEARS, seeds=seeds)


@pytest.mark.parametrize("bound", [-1, 2500, None])
def test_all_wide_and_mixed_widths(bound, monkeypatch):
    """_NARROW_MAX lowered as tests/test_sampler_compact_cpu.py does: -1 makes every block wide; at 2500 the venue
    blocks, whose venue ids are moved past it, are wide and the others narrow; at the default bound the venue blocks'
    times are moved past 2^31, which makes them wide (the time filter keeps those edges out of the sample)."""
    from pyhgt_b200 import sampler
    if bound is not None:
        monkeypatch.setattr(sampler, "_NARROW_MAX", bound)
    edges = mag_edges(P=500, A=300, Fi=40, V=20, seed=5)
    k, ei, tm = edges[3]
    if bound == 2500:
        ei = ei + torch.tensor([[3000], [0]])
    edges[3] = (k, ei, tm + (2 ** 33 if bound is None else 0))
    for placement in ("device", "host"):
        got, ref = build_both(edges, TYPES, placement)
        assert_same_graph(got, ref)
        narrow = [bool(c.skip & 2) for c in ref._cblocks]
        assert (not any(narrow)) if bound == -1 else (any(narrow) and not all(narrow))
        assert_same_batches(got, ref, "paper", YEARS)


def test_scale_ogbn_mag_sized():
    """synth.make_mag_shaped(1.0) as typed arrays: 21.1 M edges, 42.2 M with rev_; sample 32 subgraphs."""
    from pyhgt_b200 import sampler, synth
    edges, types = mag_shaped_edges()
    # times squeezed into [100, 130), so that every sampled edge's time difference fits the RTE table
    edges = [(k, ei, tm // 8 + 100) for k, ei, tm in edges]
    dg = sampler.DeviceGraph.from_edges(edges, types, _dev())
    assert dg.fg is None and dg.n_blocks == 8
    total = sum(int(a.shape[0]) for i, a in enumerate(dg._adjacency) if i % 4 == 2)
    assert 0 < total <= 2 * sum(int(e[1].shape[1]) for e in edges)
    assert all(0 < n <= c for n, c in zip(dg.n_ids, synth.MAG_NODE_COUNTS))
    rng = np.random.RandomState(0)
    inps = [{"paper": np.stack([rng.choice(dg.n_ids[0], 128, replace=False), np.full(128, 115)], 1)} for _ in range(32)]
    out = sampler.sample_subgraphs_cuda(dg, None, 3, 64, inps, torch.Generator().manual_seed(0))
    assert len(out) == 32 and all(int(o[3].shape[1]) > 0 for o in out)


def mag_shaped_edges(scale=1.0):
    """synth.make_mag_shaped(scale) split into its typed arrays (per-type ids, the edge times)."""
    from pyhgt_b200 import synth
    g = synth.make_mag_shaped(scale)
    names = ["paper", "author", "institution", "field"]
    counts = [max(2, int(round(c * scale))) for c in synth.MAG_NODE_COUNTS]
    starts = np.concatenate([[0], np.cumsum(counts)]).tolist()
    edges = []
    for r, (name, s, t, _) in enumerate(synth.MAG_RELATIONS):
        sel = g.edge_type == r
        ei = g.edge_index[:, sel] - torch.tensor([[starts[s]], [starts[t]]])
        edges.append(((names[s], name, names[t]), ei.contiguous(), g.edge_time[sel].contiguous()))
    return edges, names
