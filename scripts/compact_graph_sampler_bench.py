"""Device HGSampling from a compact graph: int64 against int32 ("narrow") adjacency blocks and fp32 against bf16 feature
tables, for a graph in device memory and one in page-locked host memory (``DeviceGraph(..., placement=...)``).

Workload: the graph and seeds of scripts/host_graph_sampler_bench.py (MAG schema, about 2.3 M edges with the reverse
relations, F = 128, 128 paper seeds per subgraph), depth 6 / width 520 and depth 3 / width 64, B = 1, 8, 32.

Per placement three graphs: "wide" (int64 blocks, fp32 tables: the layout before narrow blocks), "narrow" (int32 blocks,
fp32 tables: the default) and "bf16" (int32 blocks, bf16 tables).  The three alternate call by call, in a rotating
order, from the same generator states.  Prints one JSON line per setting, B and placement:
  ms                 ms per subgraph (CUDA events around the call / B) per graph: median, min and max over --repeats;
  narrow_over_wide   narrow median / wide median;  bf16_over_fp32: bf16 median / narrow median;
  graph_bytes        DeviceGraph.graph_bytes of each graph;
  host_read_bytes    (host placement) bytes the kernels read from host memory per subgraph, counted from the sampled
                     sizes as scripts/host_graph_sampler_bench.py counts them, at each graph's element widths;
  equal              narrow vs wide: every tensor of every member bitwise equal; bf16 vs fp32: every tensor but
                     node_feature, which equals the fp32 one rounded to bf16;
  plus the card name and power limit read in the same run.

    python scripts/compact_graph_sampler_bench.py [--scale 1.0] [--repeats 7]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from gpu_sampler_bench import F_IN, card, make_graph   # noqa: E402
from host_graph_sampler_bench import read_bytes        # noqa: E402


def frozen(g, wide):
    """FrozenGraph of g, every block int64 (wide) or in the default format (narrow wherever it fits)."""
    from pyhgt_b200 import sampler
    saved = sampler._NARROW_MAX
    try:
        if wide:
            sampler._NARROW_MAX = -1
        return sampler.FrozenGraph(g)
    finally:
        sampler._NARROW_MAX = saved


def equal(a, b, bf16=False):
    for x, y in zip(a, b):
        if bf16:
            if not torch.equal(y[0], x[0].to(torch.bfloat16).float()):
                return False
        elif not torch.equal(x[0], y[0]):
            return False
        for i in range(1, 5):
            if not torch.equal(x[i], y[i]):
                return False
        if x[5] != y[5] or list(x[7]) != list(y[7]) or any(not torch.equal(x[7][t], y[7][t]) for t in x[7]):
            return False
    return True


def stat(v):
    return {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--settings", default="6x520,3x64")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import sampler
    dev = torch.device("cuda:0")
    g, n, year, n_edges = make_graph(args.scale)
    rng = np.random.RandomState(1)
    fg0 = frozen(g, wide=True)
    tables = {t: torch.from_numpy(rng.randn(max(fg0.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    graphs = {}
    for placement in ("device", "host"):
        wide, narrow = (fg0 if placement == "device" else frozen(g, wide=True)), frozen(g, wide=False)
        graphs[placement] = {
            "wide": sampler.DeviceGraph(wide, dev, tables, placement=placement),
            "narrow": sampler.DeviceGraph(narrow, dev, tables, placement=placement),
            "bf16": sampler.DeviceGraph(narrow, dev, tables, placement=placement, feature_dtype=torch.bfloat16)}
    time_range = {y: True for y in range(1990, 2016)}
    name, power = card()

    def seeds(i):
        r = np.random.RandomState(100 + i)
        p = r.choice(np.nonzero(year <= 2015)[0], 128, replace=False)
        return {"paper": np.stack([p, year[p]], 1)}

    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        for B in (1, 8, 32):
            inps = [seeds(i) for i in range(B)]
            for placement, gs in graphs.items():
                outs = {}
                for label, dg in gs.items():               # warm-up (and the host graphs' hit scratch sizes)
                    for _ in range(2):
                        outs[label] = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps,
                                                                    torch.Generator().manual_seed(0))
                ms = defaultdict(list)
                labels = list(gs)
                for i in range(args.repeats):
                    k = i % len(labels)
                    for label in labels[k:] + labels[:k]:
                        dg = gs[label]
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        torch.cuda.synchronize()
                        e0.record()
                        sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps,
                                                      torch.Generator().manual_seed(i))
                        e1.record()
                        torch.cuda.synchronize()
                        ms[label].append(e0.elapsed_time(e1) / B)
                st = {k: stat(v) for k, v in ms.items()}
                line = {"setting": {"depth": depth, "width": width, "seeds": 128, "B": B}, "placement": placement,
                        "graph": {"nodes": n, "edges": n_edges, "feature_width": F_IN},
                        "batch_nodes_per_subgraph": int(np.mean([int(o[1].numel()) for o in outs["wide"]])),
                        "ms": st, "repeats": args.repeats,
                        "narrow_over_wide": round(st["narrow"]["median"] / st["wide"]["median"], 3),
                        "bf16_over_fp32": round(st["bf16"]["median"] / st["narrow"]["median"], 3),
                        "graph_bytes": {k: dg.graph_bytes for k, dg in gs.items()},
                        "equal": {"narrow_vs_wide": equal(outs["wide"], outs["narrow"]),
                                  "bf16_vs_fp32": equal(outs["narrow"], outs["bf16"], bf16=True)},
                        "gpu": name, "power_limit": power}
                if placement == "host":
                    rb = {}
                    for label, dg in gs.items():
                        per = [read_bytes(dg, o, width, F_IN) for o in outs[label]]
                        fe = 2 if label == "bf16" else 4
                        for p in per:                      # read_bytes counts fp32 rows
                            p["total"] += (fe - 4) * p["features"] // 4
                            p["features"] = fe * p["features"] // 4
                        rb[label] = {k: int(np.mean([p[k] for p in per])) for k in per[0]}
                    line["host_read_bytes"] = rb
                print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
