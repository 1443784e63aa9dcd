"""The c4 training step (bench.py --config c4: half of the c2 graph, 3 HGTConv(256, 256, H=8) layers, forward + backward)
with torch.use_deterministic_algorithms off and on, alternating in one process.  Prints one JSON line per round and mode:
median / min / max ms per step over CUDA-event pairs, peak memory, the per-kernel times of one profiled step (the edge
backward stages among them), and whether two steps from identical module state and inputs gave bitwise equal outputs and
gradients.  Writes nothing.

    python scripts/deterministic_train_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                # noqa: E402  (graph generator and c4 settings only)
from pyhgt_b200 import HGTConv              # noqa: E402

EDGE_BWD_KERNELS = ("k_edge_bwd", "k_edge_bwd_dst", "k_edge_bwd_rows", "k_merge_piece_rows")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    cfg = bench.CONFIGS["c4"]
    D, HEADS, L = cfg["d"], cfg["heads"], cfg["layers"]
    g = bench.make_graph("c4", args.scale)
    N, E, T, R = g.num_nodes, g.num_edges, g.num_types, g.num_relations
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([HGTConv(D, D, T, R, HEADS, 0.0, True, False) for _ in range(L)]).to(dev).train()
    HGTConv.keep_att = False
    x = torch.randn(N, D, generator=torch.Generator().manual_seed(0)).to(dev)
    w = torch.randn(N, D, generator=torch.Generator().manual_seed(1)).to(dev)
    nt, ei, et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)

    def step(keep=False):
        layers.zero_grad(set_to_none=True)
        xg = x.clone().requires_grad_(keep)
        h = xg
        for m in layers:
            h = m(h, nt, ei, et)
        (h * w).sum().backward()
        if keep:
            return [h.detach()] + [xg.grad] + [p.grad.clone() for p in layers.parameters()]
        return None

    def kernel_ms():
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        agg = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name.replace("void ", "").replace("(anonymous namespace)::", "").split("(")[0].split("<")[0]
                agg[name] = agg.get(name, 0.0) + ev.device_time_total / 1e3
        return agg

    for rnd in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
            evs[0].record()
            for i in range(args.steps):
                step()
                evs[i + 1].record()
            torch.cuda.synchronize()
            ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(args.steps))
            peak_gb = torch.cuda.max_memory_allocated() / 1e9
            a, b = step(keep=True), step(keep=True)
            differing = sum(not torch.equal(u, v) for u, v in zip(a, b))
            del a, b
            agg = kernel_ms()
            line = {"round": rnd, "deterministic": torch.are_deterministic_algorithms_enabled(),
                    "fill_uninitialized_memory": bool(torch.utils.deterministic.fill_uninitialized_memory),
                    "workload": "%s: N=%d, E=%d, d=%d, H=%d, %d layers" % (cfg["label"], N, E, D, HEADS, L),
                    "gpu": torch.cuda.get_device_name(dev), "steps": args.steps,
                    "ms_per_step": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1], "peak_mem_gb": round(peak_gb, 2),
                    "repeat_tensors": 2 + len(list(layers.parameters())), "repeat_differing": differing,
                    "edge_bwd_ms": {k: round(agg[k], 3) for k in EDGE_BWD_KERNELS if k in agg},
                    "kernel_ms_top": {k: round(v, 3) for k, v in sorted(agg.items(), key=lambda t: -t[1])[:16]}}
            print(json.dumps(line), flush=True)
    torch.use_deterministic_algorithms(False)


if __name__ == "__main__":
    main()
