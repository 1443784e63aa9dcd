"""sampler.mag_features and DeviceGraph.set_features without a GPU: the C ABI declarations, every refusal (they come
before any device work), and the rules themselves restated in numpy from the raw edge arrays against the script's
values in tests/golden/mag_features*.pt."""
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.conftest import ROOT, load_golden

DEV = torch.device("cuda:0")          # never touched
ENTRY_POINTS = ("hgt_feat_degree", "hgt_feat_neighbour_mean")


def test_header_declares_the_feature_entry_points_and_lib_binds_them():
    from pyhgt_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hgt_b200.h")).read(), flags=re.S)
    for name in ENTRY_POINTS:
        assert re.search(r"\bint %s\s*\(" % name, text), name
        assert name in _lib.SIGNATURES, name


def _graph(n_ids=(10, 7, 3)):
    """What mag_features reads before any device work: the types and their id ranges."""
    types = ["paper", "author", "institution"]
    return SimpleNamespace(types=types, n_ids=list(n_ids), slot={t: i for i, t in enumerate(types)}, device=DEV)


NUM = {"paper": 10, "author": 7, "institution": 3}


@pytest.mark.parametrize("x, num_nodes, match", [
    (torch.zeros(10, 4), {"author": 7, "institution": 3}, "'paper'"),
    (torch.zeros(9, 4), NUM, "x_paper"),
    (torch.zeros(10), NUM, "x_paper"),
    (torch.zeros(10, 4, 1), NUM, "x_paper"),
    (torch.zeros(10, 4, dtype=torch.int64), NUM, "x_paper"),
    (torch.zeros(10, 4, dtype=torch.bfloat16), NUM, "x_paper"),
    (np.zeros((10, 4), dtype=np.float32), NUM, "x_paper"),
    (torch.zeros(10, 4), {**NUM, "author": 6}, r"num_nodes\['author'\] = 6 is below"),
    (torch.zeros(9, 4), {**NUM, "paper": 9}, r"num_nodes\['paper'\] = 9 is below"),
    (torch.zeros(10, 4), {"paper": 10, "author": 7}, r"num_nodes\['institution'\] = None is below"),
])
def test_refused_arguments(x, num_nodes, match):
    from pyhgt_b200 import sampler
    with pytest.raises(ValueError, match=match):
        sampler.mag_features(_graph(), x, num_nodes)


def test_set_features_refuses_unequal_widths_before_any_device_work():
    from pyhgt_b200 import sampler
    dg = sampler.DeviceGraph.__new__(sampler.DeviceGraph)
    dg._setup(["paper", "author"], DEV, "device", None)
    with pytest.raises(ValueError, match=r"feature tables must all have the same width, got \[4, 5\]"):
        dg.set_features({"paper": torch.zeros(3, 4), "author": torch.zeros(3, 5)})


def restate_from_edges(case):
    """The script's rules in numpy from the raw arrays: per block (the key and its rev_ twin) the distinct
    (target, source) pairs; deg sums the blocks' pair counts per target; a mean sums every block's pairs."""
    nn = case["num_nodes"]
    blocks = []
    for (s_t, _, t_t), ei in case["edges"]:
        ei = ei.numpy()
        for tt, st, tgt, src in ((t_t, s_t, ei[1], ei[0]), (s_t, t_t, ei[0], ei[1])):
            pairs = np.unique(np.stack([tgt, src], 1), axis=0) if ei.shape[1] else np.zeros((0, 2), np.int64)
            blocks.append((tt, st, pairs))

    def deg(t):
        d = np.zeros(nn[t])
        for tt, _, p in blocks:
            if tt == t:
                np.add.at(d, p[:, 0], 1)
        with np.errstate(divide="ignore"):
            return np.log10(d)[:, None]

    def mean(t, s, src):
        acc, cnt = np.zeros((nn[t], src.shape[1])), np.zeros(nn[t])
        for tt, st, p in blocks:
            if (tt, st) == (t, s):
                np.add.at(acc, p[:, 0], src[p[:, 1]])
                np.add.at(cnt, p[:, 0], 1)
        return acc / np.maximum(cnt, 1)[:, None], cnt.sum()

    x = case["x_paper"].numpy().astype(np.float64)
    out = {"paper": np.concatenate([x, deg("paper")], 1)}
    author = None
    for t in nn:
        if t not in ("paper", "institution"):
            m, n = mean(t, "paper", x)
            if n:
                out[t] = np.concatenate([m, deg(t)], 1)
                author = m if t == "author" else author
    out["institution"] = np.concatenate([mean("institution", "author", author)[0], deg("institution")], 1)
    return out


@pytest.mark.parametrize("name", ["small", "mixed"])
def test_rules_restated_from_the_arrays_give_the_script_values(name):
    case = load_golden("mag_features")[name]
    ref = {t: v.numpy() for t, v in case["node_feature"].items()}
    got = restate_from_edges(case)
    assert list(got) == list(ref)
    for t in ref:
        assert got[t].shape == ref[t].shape
        assert np.array_equal(np.isinf(got[t]), np.isinf(ref[t])) and np.isinf(ref[t]).any()
        fin = np.isfinite(ref[t])
        np.testing.assert_allclose(got[t][fin], ref[t][fin], rtol=1e-12, atol=1e-14)
    # the fixture reaches the cases the rules single out
    assert any((ref["author"][:, :-1] == 0).all(1) & np.isfinite(ref["author"][:, -1]))     # an author with no paper
    (_, ei_w), (_, ei_r) = case["edges"][1], case["edges"][4]
    both = set(map(tuple, ei_w.T.tolist())) & set(map(tuple, ei_r.flip(0).T.tolist()))
    assert both and ei_w.shape[1] > len(set(map(tuple, ei_w.T.tolist())))                 # cross-key and in-key repeats
