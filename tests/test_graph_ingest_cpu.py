"""DeviceGraph.from_edges without a GPU: argument validation (every refusal comes before any kernel runs), the C ABI
declarations, and the host-side plan (block order, relation ids, row_of lengths and n_ids) against FrozenGraph on the
dict graph that the preprocessing loop builds from the same arrays."""
import os
import re

import pytest
import torch

from tests.conftest import ROOT
from tests.test_gpu_graph_ingest import TYPES, dict_graph, mag_edges

DEV = torch.device("cuda:0")          # never touched: every case below is refused, or planned, on the host
ENTRY_POINTS = ("hgt_ingest_workspace_bytes", "hgt_ingest_block_sort", "hgt_ingest_block_write")


def test_header_declares_the_ingest_entry_points_and_lib_binds_them():
    from pyhgt_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hgt_b200.h")).read(), flags=re.S)
    for name in ENTRY_POINTS:
        assert re.search(r"\bint %s\s*\(" % name, text), name
        assert name in _lib.SIGNATURES, name


def _from_edges(edges, types=("paper", "author"), **kw):
    from pyhgt_b200 import sampler
    return sampler.DeviceGraph.from_edges(edges, list(types), kw.pop("device", DEV), **kw)


def _ei(*rows):
    return torch.tensor(rows, dtype=torch.int64)


GOOD = (("author", "writes", "paper"), _ei([0, 1], [2, 3]), torch.tensor([5, 6]))


@pytest.mark.parametrize("edges, err, match", [
    ([(("author", "writes", "venue"), _ei([0], [1]), None)], KeyError, "venue"),
    ([(("x", "writes", "paper"), _ei([0], [1]), None)], KeyError, "'x'"),
    ([GOOD, GOOD], ValueError, "two keys"),
    ([GOOD, (("paper", "rev_writes", "author"), _ei([0], [1]), None)], ValueError, "two keys"),
    ([(("author", "writes"), _ei([0], [1]), None)], ValueError, "items"),
    ([("author", "writes", "paper")], ValueError, "items"),
    ([(("author", "writes", "paper"), _ei([0, 1], [2, 3], [4, 5]), None)], ValueError, r"\[2, E\]"),
    ([(("author", "writes", "paper"), _ei([0, 1]), None)], ValueError, r"\[2, E\]"),
    ([(("author", "writes", "paper"), _ei([0], [1]).int(), None)], ValueError, "int64"),
    ([(("author", "writes", "paper"), [[0], [1]], None)], ValueError, "list"),
    ([(("author", "writes", "paper"), _ei([0, 1], [2, 3]), torch.tensor([5]))], ValueError, "time"),
    ([(("author", "writes", "paper"), _ei([0, 1], [2, 3]), torch.tensor([5, 6]).int())], ValueError, "time"),
    ([(("author", "writes", "paper"), _ei([0, 1], [2, 3]), [5, 6])], ValueError, "time"),
    ([GOOD, (("paper", "cites", "paper"), _ei([0, -1], [2, 3]), None)], ValueError, "negative"),
    ([(("paper", "cites", "paper"), _ei([0, 2 ** 40], [2, 3]), None)], ValueError, "2\\^40"),
    ([(("paper", 7, "paper"), _ei([0], [1]), None)], ValueError, "str"),
])
def test_refused_input(edges, err, match):
    with pytest.raises(err, match=match):
        _from_edges(edges)


def test_refused_arguments():
    with pytest.raises(ValueError, match="placement"):
        _from_edges([GOOD], placement="disk")
    with pytest.raises(ValueError, match="feature_dtype"):
        _from_edges([GOOD], feature_dtype=torch.float16)
    with pytest.raises(ValueError, match="CUDA"):
        _from_edges([GOOD], device="cpu")
    with pytest.raises(ValueError, match="distinct"):
        _from_edges([GOOD], types=("paper", "author", "paper"))


def test_ids_below_2_40_and_non_str_relations_without_reverse_are_planned():
    from pyhgt_b200 import sampler
    keys, order = sampler._ingest_plan([(("paper", 7, "paper"), _ei([0, 2 ** 40 - 1], [2, 3]), None)],
                                       {"paper": 0}, reverse=False)
    assert order == [("paper", "paper", 7)] and keys[0]["range"] == ((0, 2 ** 40 - 1), (2, 3))


def _gapped_edges():
    g = torch.Generator().manual_seed(4)
    src = torch.randint(0, 50, (300,), generator=g) * 997 + 13
    dst = torch.randint(0, 60, (300,), generator=g) * 131 + 5
    a_src = torch.randint(0, 40, (200,), generator=g) * 50_021
    return [(("paper", "cites", "paper"), torch.stack([src, dst]), None),
            (("venue", "empty", "paper"), torch.zeros(2, 0, dtype=torch.int64), None),
            (("author", "writes", "paper"), torch.stack([a_src, dst[:200]]), None),
            (("paper", "written_by", "author"), torch.stack([dst[:100], a_src[:100] // 7]), None),
            (("paper", "self", "paper"), torch.stack([dst, dst]), None)]


@pytest.mark.parametrize("reverse", [True, False])
@pytest.mark.parametrize("case", ["mag", "gapped"])
def test_plan_matches_frozen_graph(case, reverse):
    """Block order, edge_dict, row_of lengths and n_ids of the plan equal FrozenGraph's on the dict graph."""
    from pyhgt_b200 import sampler
    edges = mag_edges(P=300, A=200, Fi=30, V=10) if case == "mag" else _gapped_edges()
    types = TYPES if case == "mag" else ["paper", "author", "venue"]
    g = dict_graph(edges, types, reverse)
    fg = sampler.FrozenGraph(g)
    keys, order = sampler._ingest_plan(edges, {t: i for i, t in enumerate(types)}, reverse)
    assert order == [(t, s, r) for t, d1 in fg.blocks.items() for s, d2 in d1.items() for r in d2]
    assert sampler._edge_dict(order) == sampler._edge_dict(g.get_meta_graph())
    row_len, n_ids = sampler._ingest_n_ids(keys, order)
    assert {t: n for t, n in n_ids.items() if n} == {t: n for t, n in fg.n_ids.items() if n}
    assert row_len == {(t, s, r): b.row_of.shape[0] for t, d1 in fg.blocks.items() for s, d2 in d1.items()
                       for r, b in d2.items()}
    if case == "gapped" and not reverse:
        # author ids reach past every author target id: the written_by block's row_of counts the writes block's
        # neighbours, which FrozenGraph met first
        assert row_len[("author", "paper", "written_by")] > int(edges[3][1][1].max()) + 1
