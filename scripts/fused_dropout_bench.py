"""Training with dropout 0.2: nn.Dropout (HGTConv.fused_dropout off) against masks drawn inside the update kernels (on).

  1. The c4 training step (3 HGTConv(256, 256, H=8) layers, use_norm, no RTE, forward + backward with every parameter's
     gradient; half of the c2 graph, bench.py --config c4) at p = 0.2: switch off and on alternate in one process, with
     the deterministic flag off and on, with and without recompute_tables.  One JSON line per round and setting: median /
     min / max ms per step over CUDA-event pairs and max_memory_allocated.
  2. The sampled ogbn-mag step of scripts/graphed_train_bench.py (GNN 128 -> 512, 4 layers, RTE, dropout 0.2, AdamW +
     OneCycleLR + clip) at depth 6 x width 520, eager and graphed, switch off and on alternating per epoch (the switch
     covers the GNN's adapter and its four layers).  One JSON line per variant.
The card's name and power limit are read in the same run.  Writes nothing.

    python scripts/fused_dropout_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0] [--epochs 3]
                                          [--mag-scale 1.0] [--no-c4] [--no-mag]
"""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench                                            # noqa: E402  (graph generator and c4 settings only)
from recompute_train_bench import hardware              # noqa: E402
from pyhgt_b200 import HGTConv                          # noqa: E402
from pyhgt_b200.model import GNN                        # noqa: E402

P_DROP = 0.2


def set_switch(module, on):
    """fused_dropout of every layer and GNN inside `module` (instance attributes: two models can differ)."""
    for m in module.modules():
        if isinstance(m, (HGTConv, GNN)):
            m.fused_dropout = on


class Stack:
    """The c4 layer stack with dropout P_DROP on one graph."""

    def __init__(self, g, dev):
        cfg = bench.CONFIGS["c4"]
        self.D, self.H, self.L = cfg["d"], cfg["heads"], cfg["layers"]
        torch.manual_seed(0)
        self.layers = torch.nn.ModuleList([HGTConv(self.D, self.D, g.num_types, g.num_relations, self.H, P_DROP, True,
                                                   False) for _ in range(self.L)]).to(dev).train()
        for m in self.layers:
            m.keep_att = False
        self.x = torch.randn(g.num_nodes, self.D, generator=torch.Generator().manual_seed(0)).to(dev)
        self.w = torch.randn(g.num_nodes, self.D, generator=torch.Generator().manual_seed(1)).to(dev)
        self.args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
        self.workload = "N=%d, E=%d, d=%d, H=%d, %d layers, dropout %g" % (g.num_nodes, g.num_edges, self.D, self.H,
                                                                          self.L, P_DROP)

    def step(self):
        self.layers.zero_grad(set_to_none=True)
        h = self.x
        for m in self.layers:
            h = m(h, *self.args)
        (h * self.w).sum().backward()

    def timed(self, fused, lean, steps, warmup):
        set_switch(self.layers, fused)
        for m in self.layers:
            m.recompute_tables = lean
        for _ in range(warmup):
            self.step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        evs[0].record()
        for i in range(steps):
            self.step()
            evs[i + 1].record()
        torch.cuda.synchronize()
        ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))
        return {"ms_per_step": round(ms[len(ms) // 2], 3), "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3),
                "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3)}


def c4_part(args, dev, hw):
    st = Stack(bench.make_graph("c4", args.scale), dev)
    label = "%s: %s" % (bench.CONFIGS["c4"]["label"], st.workload)
    for rnd in range(args.rounds):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for lean in (False, True):
                for fused in (False, True):
                    line = {"part": "c4", "round": rnd, "deterministic": det, "recompute_tables": lean,
                            "fused_dropout": fused, "workload": label, "steps": args.steps}
                    line.update(st.timed(fused, lean, args.steps, args.warmup))
                    print(json.dumps(dict(line, **hw)), flush=True)
    torch.use_deterministic_algorithms(False)


def mag_part(args, dev, hw):
    import graphed_train_bench as G
    import pyhgt_b200
    from pyhgt_b200 import graphed, plan as P, sampler
    P._CACHE_SIZE = 2 * G.BATCHES + 8
    pyhgt_b200.HGTConv.keep_att = False
    g, n, year, n_edges = G.make_graph(args.mag_scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), G.F_IN).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    paper_label = rng.randint(0, G.N_CLS, n["paper"]).astype(np.int64)
    time_range = {y: True for y in range(1990, 2016)}
    T, R = len(dg.types), len(dg.edge_dict)
    paper = dg.slot["paper"]
    depth, width = 6, 520
    batches = G.epoch_batches(dg, time_range, depth, width, year, paper_label, 0)
    sig, real = G.signature(dg, batches)
    r0 = int(sig.row0[paper])
    torch.manual_seed(0)
    base = G.Model(T, R, P_DROP).to(dev).train()
    total = (args.epochs + 1) * G.BATCHES + 1
    runs = {}
    for fused in (False, True):
        m_e, m_g = copy.deepcopy(base), copy.deepcopy(base)
        set_switch(m_e, fused)
        set_switch(m_g, fused)
        opt_e, sched_e = G.recipe(m_e, total)
        opt_g, sched_g = G.recipe(m_g, total)
        step = graphed.GraphedTrainStep(
            lambda x, nt, tm, ei, et, tg, m_g=m_g: m_g.loss(x, nt, tm, ei, et, tg[paper], r0), sig, dev, optimizer=opt_g,
            clip_norm=1.0, targets={paper: ((), torch.int64, -100)})
        runs[("eager", fused)] = lambda m=m_e, o=opt_e, s=sched_e: G.run_eager(m, o, s, batches, paper)
        runs[("graphed", fused)] = lambda st=step, s=sched_g: G.run_graphed(st, s, batches, paper)
    res = {k: [] for k in runs}
    peak = {}
    for ep in range(args.epochs + 1):                                   # epoch 0: warm-up and capture
        for k, fn in runs.items():
            torch.cuda.reset_peak_memory_stats()
            t = G.timed(fn)
            if ep:
                res[k].append(t)
                peak[k] = torch.cuda.max_memory_allocated()
    for (mode, fused), v in res.items():
        print(json.dumps(dict({"part": "mag_sampled", "mode": mode, "fused_dropout": fused,
                               "setting": {"depth": depth, "width": width, "seeds": 128, "batches_per_epoch": G.BATCHES},
                               "graph": {"nodes": n, "edges": n_edges}, "real_mean": real,
                               "padded": {"nodes": sig.n_nodes, "edges": sig.n_edges}, "epochs": args.epochs,
                               "host_ms_per_step": round(float(np.median([h for h, _ in v])), 3),
                               "event_ms_per_step": round(float(np.median([e for _, e in v])), 3),
                               "event_ms_per_step_all": [round(e, 3) for _, e in v],
                               "peak_mem_gb_process": round(peak[(mode, fused)] / 1e9, 3)}, **hw)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="c4 graph scale (1.0: half of the c2 graph)")
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--mag-scale", type=float, default=1.0)
    ap.add_argument("--no-c4", action="store_true")
    ap.add_argument("--no-mag", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    hw = hardware(dev)
    print(json.dumps(dict(hw, part="hardware")), flush=True)
    if not args.no_c4:
        c4_part(args, dev, hw)
        torch.cuda.empty_cache()
    if not args.no_mag:
        mag_part(args, dev, hw)


if __name__ == "__main__":
    main()
