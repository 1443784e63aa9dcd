"""Device HGSampling from a graph in device memory against the same graph in page-locked host memory
(``DeviceGraph(..., placement="host")``), alternating the two in one process.

Workload: the MAG-schema graph of scripts/gpu_sampler_bench.py (about 1 M edges plus reverse relations, 128-wide fp32
features), 128 paper seeds per subgraph, depth 6 / width 520 (pyHGT ogbn-mag/train_ogbn_mag.py:44-47) and depth 3 /
width 64, B = 1, 8, 32 subgraphs per ``sample_subgraphs_cuda`` call.

Prints one JSON line per setting and B:
  device_ms / host_ms   ms per subgraph (CUDA events around the call / B): median, min and max over --repeats calls,
                        device and host placement alternating call by call from the same generator states;
  host_read_bytes       bytes a host-placed graph gives the kernels per subgraph, counted from the sampled sizes:
                        add_budget (row_of + ptr of every sampled node's blocks, twice: the segment count and the draws,
                        and nbr + time of min(degree, width) neighbours), the rebuild's single read (row_of + ptr + the
                        whole nbr list of every sampled target in every block) and the feature rows;
  host_read_GBps        host_read_bytes over the host median.  Both count element bytes, so they are lower bounds on
                        link traffic: a random 8-byte read moves a whole PCIe read request;
  equal                 the two placements' batches are bitwise equal;
  plus the card name and power limit read in the same run.
With --profile, one more line per setting: CUDA kernel time per kernel name (torch.profiler) of one B = 8 call with
each placement.

    python scripts/host_graph_sampler_bench.py [--scale 1.0] [--repeats 7] [--profile]
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


def read_bytes(dg, out, width, feat_dim):
    """Bytes the kernels read from a host-placed graph for one subgraph (see the module docstring)."""
    fg = dg.fg
    indxs = out[7]
    budget = rebuild = 0
    for t, ids in indxs.items():
        ids = ids.cpu().numpy()
        for s_t, rels in fg.blocks.get(t, {}).items():
            for r, blk in rels.items():
                inside = ids[ids < blk.row_of.shape[0]]
                rows = blk.row_of[inside]
                rows = rows[rows >= 0]
                deg = blk.ptr[rows + 1] - blk.ptr[rows]
                w = blk.nbr.itemsize                  # 8, or 4 for a narrow block
                rebuild += w * inside.size + 2 * w * rows.size + w * int(deg.sum())
                if r != "self":
                    budget += 2 * (w * inside.size + 2 * w * rows.size) + 2 * w * int(np.minimum(deg, width).sum())
    feats = 4 * feat_dim * int(out[1].numel())
    return {"add_budget": budget, "rebuild": rebuild, "features": feats, "total": budget + rebuild + feats}


def same(a, b):
    for x, y in zip(a, b):
        for i in range(5):
            if not torch.equal(x[i], y[i]):
                return False
        if x[5] != y[5] or any(not torch.equal(x[7][t], y[7][t]) for t in x[7]):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--settings", default="6x520,3x64")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import sampler
    dev = torch.device("cuda:0")
    g, n, year, n_edges = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    graphs = {"device": sampler.DeviceGraph(fg, dev, tables), "host": sampler.DeviceGraph(fg, dev, tables, placement="host")}
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
            outs = {}
            for label, dg in graphs.items():                  # warm-up (and the host graph's hit scratch size)
                for _ in range(2):
                    outs[label] = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps,
                                                                torch.Generator().manual_seed(0))
            ms = defaultdict(list)
            for i in range(args.repeats):
                order = list(graphs.items()) if i % 2 == 0 else list(graphs.items())[::-1]
                for label, dg in order:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(i))
                    e1.record()
                    torch.cuda.synchronize()
                    ms[label].append(e0.elapsed_time(e1) / B)
            per = [read_bytes(graphs["host"], o, width, F_IN) for o in outs["host"]]
            rb = {k: int(np.mean([p[k] for p in per])) for k in per[0]}
            stat = {k: {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3),
                        "max": round(float(np.max(v)), 3)} for k, v in ms.items()}
            print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128, "B": B},
                              "graph": {"nodes": n, "edges": n_edges, "feature_width": F_IN},
                              "batch_nodes_per_subgraph": int(np.mean([int(o[1].numel()) for o in outs["host"]])),
                              "batch_edges_per_subgraph": int(np.mean([int(o[3].shape[1]) for o in outs["host"]])),
                              "device_ms": stat["device"], "host_ms": stat["host"], "repeats": args.repeats,
                              "host_over_device": round(stat["host"]["median"] / stat["device"]["median"], 2),
                              "host_read_bytes": rb,
                              "host_read_GBps": round(rb["total"] / stat["host"]["median"] / 1e6, 2),
                              "equal": same(outs["device"], outs["host"]),
                              "gpu": name, "power_limit": power}), flush=True)
        if args.profile:
            profile(graphs, time_range, depth, width, [seeds(i) for i in range(8)], name, power)


def profile(graphs, time_range, depth, width, inps, name, power):
    """CUDA time per kernel name of one B = 8 call per placement (a run of its own: tracing slows the host)."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    from pyhgt_b200 import sampler
    res = {}
    for label, dg in graphs.items():
        sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(0))
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(0))
            torch.cuda.synchronize()
        per = defaultdict(float)
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t:
                key = ev.key.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0]
                per[key.split("::")[-1][-40:]] += t / 1e3
        res[label] = {k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:12]}
    print(json.dumps({"profile": {"depth": depth, "width": width, "B": len(inps)}, "kernel_ms": res,
                      "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
