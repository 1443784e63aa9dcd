"""DeviceGraph.from_edges (the graph built on the device from typed edge arrays) against the dict path it replaces.

The dict path is what a user of the reference does today: the preprocessing loop (preprocess_ogbn_mag.py:29-42) fills
the 5-level edge_list dict, one insert per edge and direction, then FrozenGraph flattens it and DeviceGraph uploads it.
Graphs:
  mag_bench   the MAG schema of scripts/gpu_sampler_bench.py (paper / author / field / venue, heavy-tailed citations,
              authorship and fields; about 1 M edges with rev_) at --scale;
  ogbn_mag    synth.make_mag_shaped(1.0): ogbn-mag's four relations at full size, 21.1 M edges, 42.2 M with rev_.
Prints one JSON line per graph and placement:
  dict_s       {dict, frozen, device, total}: wall clock of the loop, FrozenGraph and DeviceGraph (ends in a device
               synchronise); "not measured" with --no-dict-at-scale on ogbn_mag;
  from_edges_s from_edges from CPU tensors to a finished graph (ends in a device synchronise), median of --repeats;
  peak_device_bytes  torch's peak allocated device memory during from_edges, above what was allocated before it;
  graph_bytes  the DeviceGraph's adjacency / feature bytes; bitwise_equal: every block array, dtype, flag, edge_dict and
  n_ids of the two graphs equal (null when the dict path was not run); plus the card name and power limit.

    python scripts/graph_ingest_bench.py [--scale 1.0] [--repeats 3] [--no-dict-at-scale]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _Graph:
    def __init__(self, edge_list, types):
        self.edge_list, self._t = edge_list, list(types)

    def get_types(self):
        return self._t

    def get_meta_graph(self):
        return [(t, s, r) for t in self.edge_list for s in self.edge_list[t] for r in self.edge_list[t][s]]


def dict_graph(edges, types):
    """The preprocessing loop: key by key, elist[t][s] = time then rlist[s][t] = time per edge, in array order."""
    el = defaultdict(lambda: defaultdict(lambda: defaultdict(lambda: defaultdict(dict))))
    for (s_t, r, t_t), ei, tm in edges:
        elist, rlist = el[t_t][s_t][r], el[s_t][t_t]["rev_" + r]
        for s_id, t_id, year in zip(ei[0].tolist(), ei[1].tolist(), tm.tolist()):
            elist[t_id][s_id] = year
            rlist[s_id][t_id] = year
    return _Graph(el, types)


def mag_bench_edges(scale, seed=0):
    """scripts/gpu_sampler_bench.py's MAG schema as typed arrays (its 'self' relations are not part of the loop)."""
    rng = np.random.RandomState(seed)
    n = {"paper": int(100000 * scale), "author": int(60000 * scale), "field": int(8000 * scale), "venue": 500}
    P = n["paper"]
    year = rng.randint(1990, 2021, P)

    def key(s_t, r, t_t, src, dst, tm):
        return (s_t, r, t_t), torch.from_numpy(np.stack([src, dst]).astype(np.int64)), torch.from_numpy(tm.astype(np.int64))

    cited = (rng.pareto(1.2, 4 * P) * 50).astype(np.int64) % P
    citing = rng.randint(0, P, 4 * P)
    pa = rng.randint(0, P, 3 * P)
    au = (rng.pareto(1.5, 3 * P) * 30).astype(np.int64) % n["author"]
    pf = rng.randint(0, P, 3 * P)
    fi = (rng.pareto(1.0, 3 * P) * 20).astype(np.int64) % n["field"]
    return [key("paper", "PP_cite", "paper", cited, citing, year[citing]),
            key("author", "AP_write", "paper", au, pa, year[pa]),
            key("field", "PF_in_L2", "paper", fi, pf, year[pf]),
            key("venue", "PV_Journal", "paper", rng.randint(0, n["venue"], P), np.arange(P), year)], list(n)


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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:                                      # noqa: BLE001
        return [torch.cuda.get_device_name(0), "not measured"]


def same_graph(a, b):
    def arr(x):
        return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    if (a.blocks, a.edge_dict, a.n_ids) != (b.blocks, b.edge_dict, b.n_ids):
        return False
    if any((x.n_row_of, x.skip, x.rel) != (y.n_row_of, y.skip, y.rel) for x, y in zip(a._cblocks, b._cblocks)):
        return False
    return all(arr(x).dtype == arr(y).dtype and np.array_equal(arr(x), arr(y)) for x, y in zip(a._adjacency, b._adjacency))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-dict-at-scale", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import sampler
    dev = torch.device("cuda:0")
    name, power = card()
    for label, (edges, types) in (("mag_bench", mag_bench_edges(args.scale)), ("ogbn_mag", mag_shaped_edges(1.0))):
        n_edges = sum(int(e[1].shape[1]) for e in edges)
        ref = None
        if label == "mag_bench" or not args.no_dict_at_scale:
            t0 = time.perf_counter()
            g = dict_graph(edges, types)
            t1 = time.perf_counter()
            fg = sampler.FrozenGraph(g)
            t2 = time.perf_counter()
            del g
            ref = sampler.DeviceGraph(fg, dev)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            dict_s = {"dict": round(t1 - t0, 2), "frozen": round(t2 - t1, 2), "device": round(t3 - t2, 2),
                      "total": round(t3 - t0, 2)}
        else:
            dict_s = "not measured"
        for placement in ("device", "host"):
            times, peak = [], 0
            for _ in range(max(1, args.repeats)):
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                t0 = time.perf_counter()
                dg = sampler.DeviceGraph.from_edges(edges, types, dev, placement=placement)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
                peak = max(peak, torch.cuda.max_memory_allocated(dev) - base)
                gb = dg.graph_bytes
                equal = same_graph(dg, ref) if ref is not None else None
                del dg
            print(json.dumps({"graph": label, "edges": n_edges, "edges_with_rev": 2 * n_edges, "placement": placement,
                              "dict_s": dict_s, "from_edges_s": round(float(np.median(times)), 3),
                              "from_edges_runs": [round(t, 3) for t in times], "peak_device_bytes": int(peak),
                              "graph_bytes": gb, "bitwise_equal": equal, "gpu": name, "power_limit": power}),
                  flush=True)
        del ref


if __name__ == "__main__":
    main()
