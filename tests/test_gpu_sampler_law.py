"""The device sampler (sample_subgraphs_cuda) against HGSampling's exact law (oracle/hgsampling_law.py), on the toy
cases of tests/test_sampler_law_cpu.py:

  * 2^18 members per case, drawn in batches of 32768 from a fixed generator seed: the true law passes a chi-square
    test at p > 1e-6 and every fault model the case can see (total variation >= 0.02) fails at p < 1e-9.  Philox is
    counter-based, so each p-value is a fixed number for a given build: the test is not flaky;
  * the weighted and the depth-2 cases run on the dense and on the hashed sampler state (the other state layouts and
    GraphedSampler are bitwise the dense path under their own tests);
  * where the law is deterministic (every budget smaller than the width) every member equals the oracle's outcome;
  * a hub of degree 5000 at width 8, where the law factorises: each of the 8 positions is uniform over the hub's
    neighbours."""
from collections import Counter

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hgsampling_law as law_mod                          # noqa: E402
from tests.test_sampler_law_cpu import CASES, law, visible_faults, _both, _graph   # noqa: E402

B = 32768                # members per call
N_DRAW = 2 ** 18         # members per case


def _dev():
    return torch.device("cuda:0")


def _device_graph(c):
    from pyhgt_b200 import sampler
    return sampler.DeviceGraph(sampler.FrozenGraph(c["graph"]), _dev())


def _outcomes(outs):
    """Each member's outcome, in the oracle's form, from one device-to-host copy of the batch's shared id and time
    buffers (every member's indxs / times are views into them)."""
    probe = next(o for o in outs if o[7])
    t0 = next(iter(probe[7]))
    lid, ntime = probe[7][t0]._base, probe[8][t0]._base
    lid_h, ntime_h = lid.cpu().numpy(), ntime.cpu().numpy()
    l0, n0 = lid.storage_offset(), ntime.storage_offset()
    got = []
    for o in outs:
        rows = []
        for t in sorted(o[7]):
            i, tm = o[7][t], o[8][t]
            a, b = i.storage_offset() - l0, tm.storage_offset() - n0
            n = i.numel()
            rows.append((t, tuple(zip(lid_h[a:a + n].tolist(), ntime_h[b:b + n].tolist()))))
        got.append(tuple(rows))
    return got


def _draw(c, layout, n, monkeypatch, seed=0, width=None):
    """Counter of the outcomes of n members (batches of B) drawn with a generator seeded by `seed`."""
    from pyhgt_b200 import plan, sampler
    dg = _device_graph(c)
    gen = torch.Generator().manual_seed(seed)
    counts = Counter()
    with monkeypatch.context() as m:
        m.setattr(sampler, "_FORCE_LAYOUT", layout)
        # the law needs the sampled nodes only: skip building a sync-free plan per member
        m.setattr(plan, "get_plan", lambda *a, **k: None)
        for k in range(0, n, B):
            outs = sampler.sample_subgraphs_cuda(dg, c["time_range"], c["depth"], width or c["width"],
                                                 [c["inp"]] * min(B, n - k), gen)
            assert dg.sampler_state["layout"] == layout
            counts.update(_outcomes(outs))
    return counts


_RUNS = [("weighted", "dense"), ("weighted", "hashed"), ("filtered", "dense"), ("cycle", "dense"),
         ("cycle", "hashed")]


@pytest.mark.parametrize("name,layout", _RUNS)
def test_device_sampler_draws_the_exact_law(name, layout, monkeypatch):
    counts = _draw(CASES[name](), layout, N_DRAW, monkeypatch, seed=1)
    assert sum(counts.values()) == N_DRAW
    p_true = law_mod.chi2_pvalue(law(name), counts)
    p_fault = {f: law_mod.chi2_pvalue(law(name, f), counts) for f in visible_faults(name)}
    print("\n%s/%s: %d outcomes seen of %d; true law p = %.4g; faults: %s" % (
        name, layout, len(counts), len(law(name)), p_true, ", ".join("%s %.3g" % kv for kv in p_fault.items())))
    assert p_true > 1e-6, p_true
    assert p_fault and all(p < 1e-9 for p in p_fault.values()), p_fault


@pytest.mark.parametrize("name", list(CASES))
def test_budgets_below_the_width_give_the_oracle_outcome_bitwise(name, monkeypatch):
    """Width 8: every adjacency and every budget is smaller than the width, so the law has one outcome (ser order and
    times), and every member must be it."""
    c = CASES[name]()
    p = law_mod.sampling_law(c["graph"], c["time_range"], c["depth"], 8, c["inp"])
    assert len(p) == 1
    (want,) = p
    counts = _draw(c, "dense", 64, monkeypatch, seed=2, width=8)
    assert list(counts) == [want]


def test_hub_positions_are_uniform(monkeypatch):
    """One paper with 5000 authors, width 8, depth 1: add_budget draws an ordered uniform 8-subset, and the budget
    (8 entries of score 1/8, count == width) is drawn as a uniform permutation of it.  So every author is included
    with probability 8 / 5000, and each position is uniform over the authors, whatever the others hold."""
    from scipy.stats import chisquare
    deg, width, n_bucket = 5000, 8, 100
    c = dict(graph=_graph(["paper", "author"], _both([(0, a, 2000) for a in range(deg)])),
             time_range={2000: True}, depth=1, width=width, inp={"paper": np.array([[0, 2000]])})
    counts = _draw(c, "dense", N_DRAW, monkeypatch, seed=3)
    ids = np.empty((N_DRAW, width), dtype=np.int64)
    r = 0
    for out, k in counts.items():
        d = dict(out)
        assert [x[0] for x in d["paper"]] == [0] and all(x[1] == 2000 for x in d["author"])
        ids[r:r + k] = [x[0] for x in d["author"]]
        r += k
    assert r == N_DRAW
    assert ids.min() >= 0 and ids.max() < deg
    assert (np.sort(ids, 1)[:, 1:] != np.sort(ids, 1)[:, :-1]).all()          # 8 distinct authors
    # inclusion: each author in 8 / 5000 of the members (about 419 expected each)
    p_incl = chisquare(np.bincount(ids.ravel(), minlength=deg)).pvalue
    # (author bucket x position): 100 buckets of 50 authors, about 2621 expected per cell
    cells = np.zeros((n_bucket, width), dtype=np.int64)
    for j in range(width):
        cells[:, j] = np.bincount(ids[:, j] * n_bucket // deg, minlength=n_bucket)
    p_cell = chisquare(cells.ravel()).pvalue
    print("\nhub: inclusion p = %.4g, bucket x position p = %.4g" % (p_incl, p_cell))
    assert p_incl > 1e-6 and p_cell > 1e-6
