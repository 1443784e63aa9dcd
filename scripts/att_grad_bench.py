"""Cost of a loss term on HGTConv.att in the c4 training step (bench.py --config c4: half of the c2 graph, 3 HGTConv(256,
256, H=8) layers, forward + backward).  Three losses alternate in one process, with torch.use_deterministic_algorithms off
and on:
    plain      (h * w).sum(), att not kept (bench.py's c4 step)
    kept       (h * w).sum() with keep_att on: att is materialised but the loss does not read it
    att        (h * w).sum() + lam * sum_l (att_l * w_att_l).sum(): the att gradient passes (hgt_edge_att_grad_prep and
               the *_att edge backward calls)
Prints one JSON line per round, mode and loss: median / min / max ms per step over CUDA-event pairs, peak memory, the
per-kernel times of the edge backward in one profiled step, and the card's name and power limit read in the same run.
Writes nothing.

    python scripts/att_grad_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0] [--lam 0.1]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                # noqa: E402  (graph generator and c4 settings only)
from pyhgt_b200 import HGTConv              # noqa: E402

EDGE_BWD_KERNELS = ("k_att_grad_prep", "k_edge_bwd", "k_edge_bwd_dst", "k_edge_bwd_rows", "k_merge_piece_rows")


def card():
    """Name, power limit and max SM clock of GPU 0, read-only query."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--lam", type=float, default=0.1)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    cfg = bench.CONFIGS["c4"]
    D, HEADS, L = cfg["d"], cfg["heads"], cfg["layers"]
    g = bench.make_graph("c4", args.scale)
    N, E, T, R = g.num_nodes, g.num_edges, g.num_types, g.num_relations
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([HGTConv(D, D, T, R, HEADS, 0.0, True, False) for _ in range(L)]).to(dev).train()
    x = torch.randn(N, D, generator=torch.Generator().manual_seed(0)).to(dev)
    w = torch.randn(N, D, generator=torch.Generator().manual_seed(1)).to(dev)
    w_att = [torch.randn(E, HEADS, generator=torch.Generator().manual_seed(2 + l)).to(dev) for l in range(L)]
    nt, ei, et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)
    gpu = card()

    def step(loss_kind):
        HGTConv.keep_att = loss_kind != "plain"
        layers.zero_grad(set_to_none=True)
        h = x
        for m in layers:
            h = m(h, nt, ei, et)
        loss = (h * w).sum()
        if loss_kind == "att":
            loss = loss + args.lam * sum((m.att * wa).sum() for m, wa in zip(layers, w_att))
        loss.backward()

    def kernel_ms(loss_kind):
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(loss_kind)
            torch.cuda.synchronize()
        agg = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name.replace("void ", "").replace("(anonymous namespace)::", "").split("(")[0].split("<")[0]
                agg[name] = agg.get(name, 0.0) + ev.device_time_total / 1e3
        return {k: round(agg[k], 3) for k in EDGE_BWD_KERNELS if k in agg}

    for rnd in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for loss_kind in ("plain", "kept", "att"):
                for _ in range(args.warmup):
                    step(loss_kind)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                evs = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
                evs[0].record()
                for i in range(args.steps):
                    step(loss_kind)
                    evs[i + 1].record()
                torch.cuda.synchronize()
                ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(args.steps))
                line = {"round": rnd, "deterministic": det, "loss": loss_kind,
                        "workload": "%s: N=%d, E=%d, d=%d, H=%d, %d layers" % (cfg["label"], N, E, D, HEADS, L),
                        "gpu": gpu, "steps": args.steps, "ms_per_step": round(ms[len(ms) // 2], 3),
                        "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3),
                        "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3),
                        "edge_bwd_ms": kernel_ms(loss_kind)}
                print(json.dumps(line), flush=True)
    torch.use_deterministic_algorithms(False)
    HGTConv.keep_att = True


if __name__ == "__main__":
    main()
