"""The device sampler's dense state (arrays over every id range) against its hashed state (per (member, type) hash tables
sized by the sample), alternating the two in one process.

Workload: the MAG-schema graph of scripts/gpu_sampler_bench.py with every node id multiplied by a stride (1, 10, 100):
the id ranges grow 10x and 100x while the graph, its degrees and the samples stay the same, which is what a graph with
sparse or very large ids looks like to the sampler.  128 paper seeds per subgraph, depth 6 / width 520 (pyHGT
ogbn-mag/train_ogbn_mag.py:44-47) and depth 3 / width 64, B = 1, 8, 32 subgraphs per ``sample_subgraphs_cuda`` call, no
features.  Then one setting past the dense state's int32 sort limit (one isolated paper seed with id 2^31 + 5 in every
member, B = 8), hashed only.

Prints one JSON line per setting:
  dense_ms / hashed_ms  ms per subgraph (CUDA events around the call / B): median, min and max over --repeats calls,
                        the two layouts alternating call by call from the same generator states;
  dense_peak_MB / hashed_peak_MB
                        peak device memory allocated during one call, above what was allocated before it;
  room / load / restarts
                        the hashed state's entries per call, its fullest region's load, and the restarts of the timed
                        calls (the warm-up calls size the room);
  rule                  the layout sample_subgraphs_cuda picks on its own for this call;
  equal                 the two layouts' batches are bitwise equal;
  plus the card name and power limit read in the same run.

    python scripts/hashed_state_sampler_bench.py [--scale 1.0] [--repeats 5]
"""
import argparse
import copy
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from gpu_sampler_bench import card, make_graph   # noqa: E402


def spread(fg, stride):
    """A copy of FrozenGraph fg whose node ids are multiplied by stride (the blocks are new, the graph dict is shared)."""
    out = copy.copy(fg)
    out.n_ids = {t: (n - 1) * stride + 1 if n else 0 for t, n in fg.n_ids.items()}
    out.blocks, out._cblocks = {}, {}
    for t_t, tes in fg.blocks.items():
        out.blocks[t_t] = {}
        for s_t, rels in tes.items():
            out.blocks[t_t][s_t] = {}
            for r, blk in rels.items():
                nb = copy.copy(blk)                  # int64 arrays whatever blk's width: spread ids may not fit int32
                nbr, tm = blk.span(0, blk.nbr.shape[0])
                nb.narrow, nb.ptr, nb.time = False, blk.ptr.astype(np.int64), tm
                nb.row_of = np.full(out.n_ids[t_t], -1, dtype=np.int64)
                nb.row_of[np.arange(blk.row_of.shape[0]) * stride] = blk.row_of
                nb.nbr = np.ascontiguousarray(nbr * stride)
                nb.nbr_addr, nb.time_addr = nb.nbr.ctypes.data, nb.time.ctypes.data
                out.blocks[t_t][s_t][r] = nb
    return out


def same(a, b):
    for x, y in zip(a, b):
        for i in range(1, 5):
            if not torch.equal(x[i], y[i]):
                return False
        if x[5] != y[5] or list(x[7]) != list(y[7]) or any(not torch.equal(x[7][t], y[7][t]) for t in x[7]):
            return False
    return True


def run(sampler, dg, layout, time_range, depth, width, inps, seed):
    """One call with the layout forced (None: the rule's choice): (batch, ms per subgraph, peak MB above the start)."""
    sampler._FORCE_LAYOUT = layout
    try:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(seed))
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1) / len(inps), (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    finally:
        sampler._FORCE_LAYOUT = None


def stat(v):
    return {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--settings", default="6x520,3x64")
    ap.add_argument("--strides", default="1,10,100")
    ap.add_argument("--batch-sizes", default="1,8,32")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import sampler
    dev = torch.device("cuda:0")
    g, n, year, n_edges = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    time_range = {y: True for y in range(1990, 2016)}
    name, power = card()

    def seeds(i, stride):
        r = np.random.RandomState(100 + i)
        p = r.choice(np.nonzero(year <= 2015)[0], 128, replace=False)
        return {"paper": np.stack([p * stride, year[p]], 1)}

    for stride in (int(s) for s in args.strides.split(",")):
        dg = sampler.DeviceGraph(spread(fg, stride) if stride > 1 else fg, dev)
        for setting in args.settings.split(","):
            depth, width = (int(v) for v in setting.split("x"))
            for B in (int(b) for b in args.batch_sizes.split(",")):
                inps = [seeds(i, stride) for i in range(B)]
                outs = {}
                for layout in ("dense", "hashed"):          # warm-up; the hashed calls size the room
                    for _ in range(2):
                        outs[layout] = run(sampler, dg, layout, time_range, depth, width, inps, 0)[0]
                ms, peak, restarts = defaultdict(list), defaultdict(float), 0
                for i in range(args.repeats):
                    order = ("dense", "hashed") if i % 2 == 0 else ("hashed", "dense")
                    for layout in order:
                        _, t, p = run(sampler, dg, layout, time_range, depth, width, inps, i)
                        ms[layout].append(t)
                        peak[layout] = max(peak[layout], p)
                        if layout == "hashed":
                            restarts += dg.sampler_state["restarts"]
                st = dict(dg.sampler_state)
                run(sampler, dg, None, time_range, depth, width, inps, 0)
                print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128, "B": B, "stride": stride},
                                  "id_ranges": dg.n_ids, "dense_ms": stat(ms["dense"]),
                                  "hashed_ms": stat(ms["hashed"]),
                                  "hashed_over_dense": round(np.median(ms["hashed"]) / np.median(ms["dense"]), 3),
                                  "dense_peak_MB": round(peak["dense"], 1), "hashed_peak_MB": round(peak["hashed"], 1),
                                  "room": st["entries"], "load": round(st["load"], 3), "restarts": restarts,
                                  "rule": dg.sampler_state["layout"], "equal": same(outs["dense"], outs["hashed"]),
                                  "repeats": args.repeats, "gpu": name, "power_limit": power}), flush=True)
        del dg
        torch.cuda.empty_cache()

    # past the dense int32 sort limit: an isolated paper seed with id 2^31 + 5 in each of 8 members
    dg = sampler.DeviceGraph(fg, dev)
    depth, width, B = 6, 520, 8
    inps = []
    for i in range(B):
        s = seeds(i, 1)
        inps.append({"paper": np.concatenate([s["paper"], [[2 ** 31 + 5, 2010]]])})
    for _ in range(2):
        run(sampler, dg, None, time_range, depth, width, inps, 0)
    ms, peak, restarts = [], 0.0, 0
    for i in range(args.repeats):
        _, t, p = run(sampler, dg, None, time_range, depth, width, inps, i)
        ms.append(t)
        peak = max(peak, p)
        restarts += dg.sampler_state["restarts"]
    print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 129, "B": B, "seed_id": 2 ** 31 + 5},
                      "rule": dg.sampler_state["layout"], "hashed_ms": stat(ms), "hashed_peak_MB": round(peak, 1),
                      "dense_state_would_need_GB": round(52 * B * (2 ** 31 + 6 + sum(dg.n_ids[1:])) / 1e9, 1),
                      "room": dg.sampler_state["entries"], "load": round(dg.sampler_state["load"], 3),
                      "restarts": restarts, "repeats": args.repeats, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
