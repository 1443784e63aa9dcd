"""Generate tests/golden/mag_features*.pt: the node features the UNMODIFIED ogbn-mag preprocessing script
(/root/reference/ogbn-mag/preprocess_ogbn_mag.py) computes, lines 1-99 of it executed as written, on small seeded
OGB-style edge sets.  TEST INFRASTRUCTURE ONLY.

Run in the dev container (the reference tree does not travel to the GPU box):
    python -m oracle.make_mag_features_golden

`ogb` is replaced by a stub whose PygNodePropPredDataset returns the seeded data object (edge_index_dict, num_nodes,
x_dict, node_year_dict), and pyHGT's plotting imports by oracle/pyg_shim.py's stand-ins.  Each case stores its inputs
(the keys in edge_index_dict order, num_nodes in its order, x_paper, the paper years) and the script's
graph.node_feature (float64 arrays, one per type it made a table for).
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import pyg_shim                      # noqa: E402
from oracle.make_golden import OUT_DIR, save_fixture   # noqa: E402

SCRIPT = os.path.join(pyg_shim.REFERENCE_ROOT, "ogbn-mag", "preprocess_ogbn_mag.py")
LAST_FEATURE_LINE = 99       # graph.node_feature['institution'] = ...; later lines are labels, splits and the dump


class _Data:
    def __init__(self, edge_index_dict, num_nodes, x_paper, years):
        self.edge_index_dict = edge_index_dict
        self.num_nodes = num_nodes
        self.x_dict = {"paper": x_paper}
        self.node_year_dict = {"paper": torch.from_numpy(years).view(-1, 1)}


def run_script(data):
    """graph.node_feature of the script's lines 1-99 run on ``data``."""
    ogb = types.ModuleType("ogb")
    npp = types.ModuleType("ogb.nodeproppred")
    npp.PygNodePropPredDataset = lambda name: [data]
    npp.Evaluator = lambda name: None
    ogb.nodeproppred = npp
    saved = {k: sys.modules.get(k) for k in ("ogb", "ogb.nodeproppred")}
    sys.modules.update({"ogb": ogb, "ogb.nodeproppred": npp})
    pyg_shim.load_reference_data()                        # reference root on sys.path, plotting stand-ins
    with open(SCRIPT) as f:
        lines = f.read().splitlines()[:LAST_FEATURE_LINE]
    code = compile("\n".join(lines) + "\n", SCRIPT, "exec")
    ns = {"__name__": "preprocess_ogbn_mag", "Evaluator": npp.Evaluator}    # line 20 uses it without an import
    argv = sys.argv
    try:
        sys.argv = [SCRIPT]
        with contextlib.redirect_stdout(io.StringIO()), np.errstate(divide="ignore"):   # log10(0) = -inf is a rule
            exec(code, ns)
    finally:
        sys.argv = argv
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return {t: np.asarray(v, dtype=np.float64) for t, v in ns["graph"].node_feature.items()}


def _pairs(rng, n, lo_hi_s, lo_hi_t):
    return np.stack([rng.randint(*lo_hi_s, n), rng.randint(*lo_hi_t, n)]).astype(np.int64)


def make_case(seed, P, A, I, Fo, F, extra, wide_years=False, empty_venue=False):
    """An ogbn-mag-like edge set.  Ids leave ``extra`` nodes of each type without edges (num_nodes above the largest
    id); author A - 1 only has an institution; one (author, paper) pair repeats inside 'writes' and also appears as a
    ('paper', 'reviewed_by', 'author') pair, so the author-paper blocks hold it twice; with ``wide_years`` half the
    papers have years past 2^31, which makes the blocks whose times come from them int64; with ``empty_venue`` an empty
    ('paper', 'in', 'venue') key gives venue paper blocks without pairs (the script makes it no table)."""
    rng = np.random.RandomState(seed)
    years = rng.randint(2000, 2020, P + extra).astype(np.int64)
    if wide_years:
        years[::2] += 2 ** 33
    writes = _pairs(rng, 4 * P, (0, A - 1), (0, P))
    writes = np.concatenate([writes, writes[:, :5], [[A - 2], [P - 1]]], 1)          # repeats inside the key
    reviewed = np.concatenate([_pairs(rng, P // 2, (0, P), (0, A - 1)), writes[::-1, :3]], 1)
    affil = np.concatenate([_pairs(rng, A, (0, A), (0, I)), [[A - 1], [I - 1]]], 1)
    cites = _pairs(rng, 3 * P, (0, P), (0, P))
    topic = _pairs(rng, 2 * P, (0, P), (0, Fo))
    edges = [(("author", "affiliated_with", "institution"), affil),
             (("author", "writes", "paper"), writes),
             (("paper", "cites", "paper"), cites),
             (("paper", "has_topic", "field_of_study"), topic),
             (("paper", "reviewed_by", "author"), reviewed)]
    num_nodes = {"author": A + extra, "field_of_study": Fo + extra, "institution": I + extra, "paper": P + extra}
    if empty_venue:
        edges.append((("paper", "in", "venue"), np.zeros((2, 0), dtype=np.int64)))
        num_nodes["venue"] = 4
    x = torch.from_numpy(rng.randn(P + extra, F).astype(np.float32))
    edge_index_dict = {k: torch.from_numpy(np.ascontiguousarray(ei)) for k, ei in edges}
    feats = run_script(_Data(edge_index_dict, num_nodes, x, years))
    return {"edges": [(k, ei.clone()) for k, ei in edge_index_dict.items()], "num_nodes": dict(num_nodes),
            "x_paper": x, "years": torch.from_numpy(years), "node_feature": {t: torch.from_numpy(v) for t, v in feats.items()}}


def main():
    os.makedirs(OUT_DIR, exist_ok=True)
    fx = {
        # F = 128 as OGB's x_paper
        "small": make_case(41, P=160, A=120, I=12, Fo=25, F=128, extra=6),
        # F = 37 (not a multiple of 4: the scalar gather, two column tiles), years past 2^31 (mixed block widths),
        # a type the script makes no table for
        "mixed": make_case(42, P=120, A=90, I=9, Fo=14, F=37, extra=3, wide_years=True, empty_venue=True),
    }
    for name, case in fx.items():
        print("%-6s %s" % (name, {t: tuple(v.shape) for t, v in case["node_feature"].items()}))
    size = save_fixture(fx, "mag_features")
    print("mag_features  %.0f KB" % (size / 1024))


if __name__ == "__main__":
    main()
