"""HGSampling's exact output law (oracle/hgsampling_law.py) on toy graphs, without a GPU:

  * the oracle is well formed: every law sums to 1, and successive sampling equals a brute-force enumeration of
    numpy's draw-with-replacement loop;
  * the oracle is the reference's law: the host sampler, which replays the reference's numpy stream bit for bit
    (tests/test_sampler.py), passes a chi-square test against it on every case;
  * the cases have power: every fault model of oracle/hgsampling_law.py is at least 0.02 away in total variation from
    the true law on some case, so tests/test_gpu_sampler_law.py can tell a wrong device sampler from a right one.

Total-variation distance from the true law, per case and fault model ('-': no difference):

    fault               weighted  filtered     cycle
    weight_s               0.354         -     0.060
    weight_s3              0.278         -     0.048
    uniform_select         0.695         -     0.125
    ge_width                   -         -     0.167
    first_writer_time          -         -     0.396
    filter_ge                  -     0.600     0.297
    none_time_max              -     0.600         -
    subset_sorted              -     0.300         -
    score_by_degree            -         -     0.118
    type_order_fixed           -         -     0.973
    no_exclusion               -         -     0.717

ge_width leaves the filtered case's law alone: there the budget's entries have equal scores, and a uniform permutation
of a uniformly ordered draw is the draw's own law.

The hub case (one paper with 5000 authors, width 8) is not enumerated: its law factorises, and the GPU test checks it
in closed form."""
import functools
from collections import Counter, defaultdict

import numpy as np
import pytest

from oracle import hgsampling_law as law_mod

N_HOST = 20000           # host draws per case


class _Stub:
    def __init__(self, edge_list, types, meta):
        self.edge_list, self._t, self._m = edge_list, types, meta

    def get_types(self):
        return self._t

    def get_meta_graph(self):
        return self._m


def _graph(types, edges):
    """A dict graph from (target_type, source_type, relation, target_id, source_id, time) rows, in row order; a
    relation and its reverse are listed separately."""
    el = defaultdict(lambda: defaultdict(lambda: defaultdict(dict)))
    meta = []
    for t_t, s_t, r, tid, sid, tm in edges:
        el[t_t][s_t][r].setdefault(tid, {})[sid] = tm
        if (t_t, s_t, r) not in meta:
            meta.append((t_t, s_t, r))
    return _Stub(el, list(types), meta)


def _both(rows):
    """paper <-> author rows (paper, author, time) as AP_write and rev_AP_write edges."""
    out = []
    for p, a, tm in rows:
        out.append(("paper", "author", "AP_write", p, a, tm))
    for p, a, tm in rows:
        out.append(("author", "paper", "rev_AP_write", a, p, tm))
    return out


def case_weighted():
    """Depth 1, width 4: five seed papers with fewer authors than the width, so the budget is fixed: seven authors
    with scores 3/2, 1, 5/6, 2/3, 1/3, 1/3, 1/3 (weights s^2 from 2.25 down to 1/9, twenty times below the top), in
    insertion order a0..a6.  Count 7 > 4: one weighted draw of an ordered 4-subset."""
    rows = [(0, 0, 2000),
            (1, 0, 2000), (1, 1, 2000),
            (2, 1, 2000), (2, 2, 2000),
            (3, 2, 2000), (3, 3, 2000), (3, 4, 2000),
            (4, 3, 2000), (4, 5, 2000), (4, 6, 2000)]
    g = _graph(["paper", "author"], _both(rows))
    inp = {"paper": np.array([[p, 2000] for p in range(5)])}
    return dict(graph=g, time_range={2000: True, 2001: True}, depth=1, width=4, inp=inp)


def case_filtered():
    """Depth 1, width 3: one seed paper (time 2000) with five authors, max time 2001.  Edge times: a0 2000, a1 2002
    (past the range), a2 None (the seed's time), a3 2001 (on the bound), a4 1999.  The draw of an ordered 3-subset
    keeps 2 or 3 authors: with 2 the budget is smaller than the width and its insertion order (the draw order) is the
    sample's order, with 3 it is a uniform permutation."""
    rows = [(0, 0, 2000), (0, 1, 2002), (0, 2, None), (0, 3, 2001), (0, 4, 1999)]
    g = _graph(["paper", "author"], _both(rows))
    inp = {"paper": np.array([[0, 2000]])}
    return dict(graph=g, time_range={1999: True, 2001: True}, depth=1, width=3, inp=inp)


def case_cycle():
    """Depth 2, width 2, on author <-> paper with citations; the graph's type order is (author, paper).  The seed
    author a0 has three papers: an ordered 2-subset of them enters the budget.  Layer 1 selects both (count == width,
    a uniform permutation) and their add_budget excludes a0, gives a1 two writers with different times (the last one
    sets its time), and touches the author budget for the first time, mid-walk; p0 cites p3, which becomes the paper
    budget.  Layer 2 walks paper before author (first-touch order): p3 joins and its authors add to the author budget
    (p3 has three authors, more than the width, so its subset scores 1/2 each, not 1/3) before the authors are
    drawn."""
    ap = [(0, 0, 2000), (0, 1, 2001), (0, 2, 2001),
          (1, 0, 2000), (1, 1, 1999),
          (2, 0, 2000), (2, 3, 2000),
          (3, 2, 2000), (3, 4, 1998), (3, 5, 2000)]
    cite = [("paper", "paper", "cite", 0, 3, 2000), ("paper", "paper", "rev_cite", 3, 0, 2000)]
    g = _graph(["author", "paper"], _both(ap) + cite)
    inp = {"author": np.array([[0, 2000]])}
    return dict(graph=g, time_range={1998: True, 2001: True}, depth=2, width=2, inp=inp)


CASES = {"weighted": case_weighted, "filtered": case_filtered, "cycle": case_cycle}

# (case, fault) pairs the cases must tell apart: total variation >= 0.02 (module docstring's table)
MIN_TV = 0.02


@functools.lru_cache(maxsize=None)
def law(name, fault=None):
    """The law of case `name` (under a fault model), computed once per process."""
    c = CASES[name]()
    return law_mod.sampling_law(c["graph"], c["time_range"], c["depth"], c["width"], c["inp"], fault)


def visible_faults(name):
    """The fault models case `name` separates from the true law by at least MIN_TV."""
    return [f for f in law_mod.FAULTS if law_mod.total_variation(law(name), law(name, f)) >= MIN_TV]


# ---- the oracle is well formed ---------------------------------------------------------------------------------

@pytest.mark.parametrize("fault", [None] + list(law_mod.FAULTS))
@pytest.mark.parametrize("name", list(CASES))
def test_every_law_sums_to_one(name, fault):
    p = law(name, fault)
    assert abs(sum(p.values()) - 1.0) < 1e-12
    assert all(v > 0 for v in p.values())
    assert len(p) <= 5000


def _first_distinct_law(weights, k, length):
    """Brute force of numpy's legacy choice(p=w, replace=False): every i.i.d. sequence of `length` draws from w,
    mapped to its first k distinct values in order of appearance.  Returns (law, mass of sequences with fewer than k)."""
    n = len(weights)
    p = np.asarray(weights, dtype=np.float64) / np.sum(weights)
    seqs = np.array(np.meshgrid(*[np.arange(n)] * length, indexing="ij")).reshape(length, -1).T
    prob = np.prod(p[seqs], axis=1)
    out, short = defaultdict(float), 0.0
    for s, q in zip(seqs.tolist(), prob.tolist()):
        first = tuple(dict.fromkeys(s))[:k]
        if len(first) < k:
            short += q
        else:
            out[first] += q
    return out, short


@pytest.mark.parametrize("weights,k,length", [([1.0, 2.0, 3.0], 2, 9), ([0.5, 0.25, 1.0, 2.0], 2, 9),
                                              ([3.0, 1.0, 2.0, 2.0], 3, 9), ([2.0, 2.0, 1.0, 0.1], 1, 7)])
def test_successive_sampling_equals_brute_force(weights, k, length):
    exact = law_mod.successive_law(weights, k)
    brute, short = _first_distinct_law(weights, k, length)
    assert abs(sum(exact.values()) - 1.0) < 1e-12
    assert set(brute) == set(exact)
    for key, v in exact.items():
        # the truncated sequences miss at most `short` of each outcome's mass
        assert brute[key] <= v + 1e-12 and v - brute[key] <= short + 1e-12, key
    assert short < 0.035


def test_uniform_subset_law():
    p = law_mod.successive_law([1.0] * 5, 3)
    assert len(p) == 60 and max(abs(v - 1 / 60) for v in p.values()) < 1e-15


def test_faults_change_the_law_only_where_they_apply():
    """A fault model that does not touch any rule a case exercises leaves its law exactly as it is: each model
    changes one rule and nothing else."""
    for name in CASES:
        for fault in law_mod.FAULTS:
            if fault not in visible_faults(name):
                assert law_mod.total_variation(law(name), law(name, fault)) < 1e-12, (name, fault)


# ---- the oracle is the reference's law ---------------------------------------------------------------------------

def host_outcome(indxs, times):
    return tuple((t, tuple(zip(map(int, indxs[t]), map(int, times[t])))) for t in sorted(indxs) if len(indxs[t]))


@pytest.mark.parametrize("name", list(CASES))
def test_host_sampler_draws_the_oracle_law(name):
    from pyhgt_b200 import sampler
    from tests.test_sampler import _extractor
    c = CASES[name]()
    fg = sampler.FrozenGraph(c["graph"])
    counts = Counter()
    for s in range(N_HOST):
        np.random.seed(s)
        _, times, _, indxs, _ = sampler.sample_subgraph(fg, c["time_range"], c["depth"], c["width"], c["inp"],
                                                        _extractor)
        counts[host_outcome(indxs, times)] += 1
    assert law_mod.chi2_pvalue(law(name), counts) > 1e-6


# ---- the cases have power ----------------------------------------------------------------------------------------

def test_every_fault_is_visible_in_some_case():
    seen = {f: max(law_mod.total_variation(law(n), law(n, f)) for n in CASES) for f in law_mod.FAULTS}
    assert all(v >= MIN_TV for v in seen.values()), seen


def test_a_single_bad_outcome_or_a_skewed_sample_is_rejected():
    """The chi-square helper itself: an outcome of probability zero rejects; a sample drawn from a fault law at the
    host test's size is rejected against the true law."""
    p = law("weighted")
    rng = np.random.RandomState(0)
    keys = list(p)
    good = Counter(keys[i] for i in rng.choice(len(keys), N_HOST, p=np.array([p[k] for k in keys])))
    assert law_mod.chi2_pvalue(p, good) > 1e-6
    assert law_mod.chi2_pvalue(p, good + Counter({(("author", ((99, 0),)),): 1})) == 0.0
    q = law("weighted", "uniform_select")
    qk = list(q)
    bad = Counter(qk[i] for i in rng.choice(len(qk), N_HOST, p=np.array([q[k] for k in qk])))
    assert law_mod.chi2_pvalue(p, bad) < 1e-9
