"""The exact output law of HGSampling (pyHGT/data.py:87-175) on small graphs, in float64.  TEST INFRASTRUCTURE ONLY.

``sampling_law`` restates the reference's budget process over a dict graph (``edge_list[target_type][source_type]
[relation][target_id][source_id] = time``) and enumerates every way its random calls can go, by depth-first replay:
the process is re-run with a prefix of choices and branches at the first choice the prefix does not fix.  The result
maps each outcome to its probability.  An outcome is a tuple ``((type, ((id, time), ...)), ...)``: per sampled type
(sorted by name) the ``layer_data`` entries in ser order, seeds included.

The process has two random calls, and both are successive sampling without replacement (``successive_law``): pick
one index with probability w_i / (sum of the weights not yet picked), remove it, repeat k times.  An ordered outcome
(i_1, ..., i_k) has probability prod_j w_{i_j} / (W - sum_{l<j} w_{i_l}).

* ``np.random.choice(keys, k, replace=False)`` in ``add_budget`` (taken when ``len(adl) >= k``) is
  ``permutation(n)[:k]``: a uniform ordered k-subset, successive sampling with equal weights, each outcome of
  probability 1 / (n (n-1) ... (n-k+1)).
* ``np.random.choice(n, k, p=score, replace=False)`` in the layer loop, weights s^2.  numpy's legacy loop draws with
  replacement from p, keeps the first occurrence of each index, zeroes the found ones and redraws the shortfall.  In
  law that is one i.i.d. stream from p with repeats discarded.  Given the first j picks, whose weights sum to S_j, the
  next new index is i with probability sum_{r>=0} (S_j / W)^r w_i / W = w_i / (W - S_j): successive sampling.
* The device sampler sorts Efraimidis-Spirakis keys log(u_i) / w_i in descending order.  -log(u_i) / w_i is
  exponential with rate w_i, so the smallest is i with probability w_i / W.  By memorylessness the others, less that
  minimum, are again independent exponentials with the same rates, so the rest of the order is the same law on the
  remaining indices: successive sampling again.

Every rule the device sampler must match lives in ``_replay``: the strict ``>`` time filter, a None edge time taken as
the target's time, the exclusion of sources already in ``layer_data``, ``+= 1 / len(sampled_ids)``, the last writer
setting the budget time, the whole budget in insertion order when ``sampled_number > len(keys)``, the budget's types
walked in first-touch order, and ``budget.pop``.

``FAULTS`` names models of a wrong sampler, each of which changes exactly one of those rules; ``sampling_law(...,
fault=name)`` is that sampler's law.  The tests use them to show that a case can tell a wrong sampler from the right
one.
"""
from collections import defaultdict

FAULTS = {
    "weight_s": "select with weight s instead of s^2",
    "weight_s3": "select with weight s^3 instead of s^2",
    "uniform_select": "selection ignores the scores",
    "ge_width": "the whole budget in insertion order also when its size equals the width",
    "first_writer_time": "the first writer of a budget entry sets its time",
    "filter_ge": "the time filter drops times >= the maximum instead of > it",
    "none_time_max": "a None edge time becomes the time range's maximum instead of the target's time",
    "subset_sorted": "a neighbour subset is taken in adjacency order, not in draw order",
    "score_by_degree": "a candidate's score grows by 1 / degree instead of 1 / len(sampled_ids)",
    "type_order_fixed": "the budget's types are walked in the graph's type order instead of first-touch order",
    "no_exclusion": "sources already sampled are not excluded from the budget",
}


def successive_law(weights, k):
    """{ordered index tuple: probability} of successive sampling of k indices without replacement (module docstring)."""
    law = {}

    def walk(prefix, prob, left):
        if len(prefix) == k:
            law[prefix] = law.get(prefix, 0.0) + prob
            return
        total = sum(weights[i] for i in left)
        for i in left:
            if weights[i] > 0:
                walk(prefix + (i,), prob * weights[i] / total, [j for j in left if j != i])

    walk((), 1.0, list(range(len(weights))))
    return law


class _Branch(Exception):
    def __init__(self, options):
        super().__init__()
        self.options = options                  # [(index, probability)]


class _Tape:
    """The choices of one replay: each pick is read from the prefix, or raises _Branch with its options."""

    def __init__(self, prefix):
        self.prefix, self.pos = prefix, 0

    def successive(self, weights, k):
        picked = []
        for _ in range(k):
            if self.pos < len(self.prefix):
                picked.append(self.prefix[self.pos])
                self.pos += 1
                continue
            left = [i for i in range(len(weights)) if i not in picked and weights[i] > 0]
            total = sum(weights[i] for i in left)
            raise _Branch([(i, weights[i] / total) for i in left])
        return picked


def _replay(graph, types, time_range, depth, width, inp, tape, fault):
    max_time = max(time_range) if time_range is not None else None
    layer_data = defaultdict(dict)              # type -> {id: [ser, time]}
    budget = {}                                 # type -> {id: [score, time]}, both in first-touch order

    def add_budget(te, target_id, target_time):
        for source_type, tes in te.items():
            for relation, tesr in tes.items():
                if relation == "self" or target_id not in tesr:
                    continue
                adl = tesr[target_id]
                keys = list(adl.keys())
                if len(keys) < width:
                    sampled = keys
                else:
                    picks = tape.successive([1.0] * len(keys), width)
                    if fault == "subset_sorted":
                        picks = sorted(picks)
                    sampled = [keys[i] for i in picks]
                for source_id in sampled:
                    source_time = adl[source_id]
                    if source_time is None:
                        source_time = max_time if fault == "none_time_max" else target_time
                    if max_time is not None:
                        late = source_time >= max_time if fault == "filter_ge" else source_time > max_time
                        if late:
                            continue
                    if fault != "no_exclusion" and source_id in layer_data[source_type]:
                        continue
                    entries = budget.setdefault(source_type, {})
                    new = source_id not in entries
                    entry = entries.setdefault(source_id, [0.0, 0])
                    entry[0] += 1.0 / (len(keys) if fault == "score_by_degree" else len(sampled))
                    if new or fault != "first_writer_time":
                        entry[1] = source_time

    for _type in inp:
        for _id, _time in inp[_type]:
            layer_data[_type][_id] = [len(layer_data[_type]), _time]
    for _type in inp:
        for _id, _time in inp[_type]:
            add_budget(graph.edge_list.get(_type, {}), _id, _time)

    for _layer in range(depth):
        sts = list(budget.keys())
        if fault == "type_order_fixed":
            sts = [t for t in types if t in budget]
        for source_type in sts:
            te = graph.edge_list.get(source_type, {})
            entries = budget[source_type]
            keys = list(entries.keys())
            if width > len(keys) or (fault == "ge_width" and width == len(keys)):
                sampled = keys
            else:
                s = [entries[k][0] for k in keys]
                if fault == "uniform_select":
                    w = [1.0] * len(s)
                else:
                    e = {"weight_s": 1, "weight_s3": 3}.get(fault, 2)
                    w = [v ** e for v in s]
                sampled = [keys[i] for i in tape.successive(w, width)]
            for k in sampled:
                layer_data[source_type][k] = [len(layer_data[source_type]), entries[k][1]]
            for k in sampled:
                add_budget(te, k, entries[k][1])
                entries.pop(k)

    out = []
    for t in sorted(layer_data):
        rows = sorted(layer_data[t].items(), key=lambda kv: kv[1][0])
        if rows:
            out.append((t, tuple((int(i), int(v[1])) for i, v in rows)))
    return tuple(out)


def sampling_law(graph, time_range, sampled_depth, sampled_number, inp, fault=None):
    """{outcome: float64 probability} of ``sample_subgraph(graph, time_range, sampled_depth, sampled_number, inp)``
    (``fault``: None, or a name in FAULTS).  ``graph`` has ``edge_list`` and ``get_types()``; ``time_range`` None
    turns the time filter off, as the device sampler's does.  Exponential in the number of draws: small graphs only."""
    if fault is not None and fault not in FAULTS:
        raise ValueError("unknown fault model %r" % (fault,))
    types = list(graph.get_types())
    law = defaultdict(float)
    stack = [((), 1.0)]
    while stack:
        prefix, prob = stack.pop()
        try:
            out = _replay(graph, types, time_range, sampled_depth, sampled_number, inp, _Tape(prefix), fault)
        except _Branch as b:
            stack.extend((prefix + (i,), prob * p) for i, p in b.options)
            continue
        law[out] += prob
    return dict(law)


def total_variation(p, q):
    return 0.5 * sum(abs(p.get(k, 0.0) - q.get(k, 0.0)) for k in set(p) | set(q))


def chi2_pvalue(law, counts):
    """p-value of a chi-square goodness-of-fit test of observed outcome counts ({outcome: count}) against ``law``.
    Outcomes are pooled, least likely first, into bins of at least 5 expected draws.  An observed outcome the law
    gives probability zero rejects outright (p = 0)."""
    import numpy as np
    from scipy.stats import chisquare
    n = sum(counts.values())
    if any(k not in law or law[k] <= 0.0 for k in counts if counts[k]):
        return 0.0
    keys = sorted(law, key=lambda k: (law[k], repr(k)))
    exp, obs = [], []
    e_acc = o_acc = 0.0
    for k in keys:
        e_acc += law[k] * n
        o_acc += counts.get(k, 0)
        if e_acc >= 5.0:
            exp.append(e_acc)
            obs.append(o_acc)
            e_acc = o_acc = 0.0
    if e_acc or o_acc:
        if exp:
            exp[-1] += e_acc
            obs[-1] += o_acc
        else:
            exp.append(e_acc)
            obs.append(o_acc)
    if len(exp) < 2:
        return 1.0
    exp = np.asarray(exp)
    return float(chisquare(np.asarray(obs, dtype=np.float64), exp * (n / exp.sum())).pvalue)
