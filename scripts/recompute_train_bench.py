"""HGTConv.recompute_tables on the c4 training step (3 HGTConv(256, 256, H=8) layers, use_norm, no RTE, dropout 0,
forward + backward with every parameter's gradient), and the same step on the whole ogbn-mag-shaped graph in lean mode.

  1. c4 (half of the c2 graph, bench.py --config c4): keep and lean alternate in one process, with the deterministic
     flag off and on; one JSON line per round, flag and mode: median / min / max ms per step over CUDA-event pairs and
     max_memory_allocated.
  2. Gradients of keep and lean from identical module state and inputs: bitwise equal with the flag on; max-abs and
     relative Frobenius difference with it off.
  3. The full c2 graph (synth.make_mag_shaped(1.0)) in lean mode only (the keep mode does not fit on an 80 GB H100):
     ms per step and peak memory.
The card's name and power limit are read in the same run.  Writes nothing.

    python scripts/recompute_train_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0] [--no-full]
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
from pyhgt_b200 import HGTConv, synth       # noqa: E402


def hardware(dev):
    line = {"gpu": torch.cuda.get_device_name(dev)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
        line["power_limit_and_max_sm_clock"] = out
    except (OSError, subprocess.SubprocessError) as e:
        line["power_limit_and_max_sm_clock"] = "unavailable: %s" % e
    return line


class Stack:
    """The c4 layer stack on one graph."""

    def __init__(self, g, dev):
        cfg = bench.CONFIGS["c4"]
        self.D, self.H, self.L = cfg["d"], cfg["heads"], cfg["layers"]
        torch.manual_seed(0)
        self.layers = torch.nn.ModuleList([HGTConv(self.D, self.D, g.num_types, g.num_relations, self.H, 0.0, True, False)
                                           for _ in range(self.L)]).to(dev).train()
        for m in self.layers:
            m.keep_att = False
        self.x = torch.randn(g.num_nodes, self.D, generator=torch.Generator().manual_seed(0)).to(dev)
        self.w = torch.randn(g.num_nodes, self.D, generator=torch.Generator().manual_seed(1)).to(dev)
        self.args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
        self.workload = "N=%d, E=%d, d=%d, H=%d, %d layers" % (g.num_nodes, g.num_edges, self.D, self.H, self.L)

    def step(self, lean, keep=False):
        for m in self.layers:
            m.recompute_tables = lean
        self.layers.zero_grad(set_to_none=True)
        h = self.x
        for m in self.layers:
            h = m(h, *self.args)
        (h * self.w).sum().backward()
        if keep:
            return [h.detach()] + [p.grad.clone() for p in self.layers.parameters()]
        return None

    def timed(self, lean, steps, warmup):
        for _ in range(warmup):
            self.step(lean)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        evs[0].record()
        for i in range(steps):
            self.step(lean)
            evs[i + 1].record()
        torch.cuda.synchronize()
        ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))
        return {"ms_per_step": round(ms[len(ms) // 2], 3), "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3),
                "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="c4 graph scale (1.0: half of the c2 graph)")
    ap.add_argument("--full-scale", type=float, default=1.0, help="graph scale of the lean-only run (1.0: c2)")
    ap.add_argument("--no-full", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    hw = hardware(dev)
    print(json.dumps(dict(hw, part="hardware")), flush=True)

    st = Stack(bench.make_graph("c4", args.scale), dev)
    label = "%s: %s" % (bench.CONFIGS["c4"]["label"], st.workload)
    for rnd in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for lean in (False, True):
                line = {"part": "c4", "round": rnd, "deterministic": det, "mode": "lean" if lean else "keep",
                        "workload": label, "steps": args.steps}
                line.update(st.timed(lean, args.steps, args.warmup))
                print(json.dumps(line), flush=True)
    for det in (True, False):
        torch.use_deterministic_algorithms(det)
        keep, lean = st.step(False, keep=True), st.step(True, keep=True)
        names = ["out"] + [n for n, _ in st.layers.named_parameters()]
        line = {"part": "gradients", "deterministic": det, "workload": label, "tensors": len(names),
                "bitwise_equal": sum(torch.equal(a, b) for a, b in zip(keep, lean))}
        if not det:
            rel = {n: (b.double() - a.double()).norm().item() / max(a.double().norm().item(), 1e-30)
                   for n, a, b in zip(names, keep, lean)}
            line["max_abs"] = max((b - a).abs().max().item() for a, b in zip(keep, lean))
            line["max_rel_fro"] = max(rel.values())
            line["worst"] = max(rel, key=rel.get)
        print(json.dumps(line), flush=True)
        del keep, lean
    torch.use_deterministic_algorithms(False)
    del st
    torch.cuda.empty_cache()

    if not args.no_full:
        g = synth.make_mag_shaped(args.full_scale)
        st = Stack(g, dev)
        line = {"part": "full_graph_lean", "mode": "lean", "deterministic": False,
                "workload": "ogbn-mag-shaped x%g (c2), 3-layer stack fwd+bwd: %s" % (args.full_scale, st.workload),
                "steps": args.steps}
        line.update(st.timed(True, args.steps, args.warmup))
        print(json.dumps(dict(line, **hw)), flush=True)


if __name__ == "__main__":
    main()
