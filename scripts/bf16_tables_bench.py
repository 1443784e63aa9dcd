"""HGT layers with fp32 and bf16 gather tables ([K'|V'] and RTE), alternating autocast off / bf16 in one process.  Prints
one JSON line per round, config and mode:
  c2 / c3 / c5 forward (one HGTConv, bench.py's graphs and widths): median CUDA-event ms per forward, the `edge` and
      `proj_linear` stage times from HGTConv.event_sink, the edge kernel's algorithmic bytes (s_kv = 4 or 2) and GB/s, and
      the max-abs / relative-Frobenius deviation of the output from the fp32 output on the same seeded inputs;
  c4 training step (3 layers, forward + backward): median ms per step and max_memory_allocated.
The card name and power limit are read in the same run.  Writes nothing.

    python scripts/bf16_tables_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                # noqa: E402  (graph generator and config settings only)
from pyhgt_b200 import HGTConv              # noqa: E402


def edge_bytes(n_edges, n_dst, d, rte, s_kv):
    """E * (2 d s_kv [K'|V' row] + 4 [kv_row] (+ 4 [rte_row])) + N_dst * (d*4 [Q] + d*4 [agg] + 4 [row_ptr])."""
    return n_edges * (2 * d * s_kv + 4 + (4 if rte else 0)) + n_dst * (2 * d * 4 + 4)


def _autocast(bf16):
    return torch.autocast("cuda", dtype=torch.bfloat16) if bf16 else contextlib.nullcontext()


def _card(dev):
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index or 0)],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = None
    return torch.cuda.get_device_name(dev), pl


def forward_lines(config, scale, steps, warmup, rnd, dev, card):
    cfg = bench.CONFIGS[config]
    d, H, rte = cfg["d"], cfg["heads"], cfg["rte"]
    g = bench.make_graph(config, scale)
    N, E, T, R = g.num_nodes, g.num_edges, g.num_types, g.num_relations
    torch.manual_seed(0)
    m = HGTConv(d, d, T, R, H, 0.0, True, rte).to(dev).eval()
    m.keep_att = False
    x = torch.randn(N, d, generator=torch.Generator().manual_seed(0)).to(dev)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev) if rte else None)
    n_dst = int((torch.bincount(g.edge_index[1], minlength=N) > 0).sum())
    outs = {}
    for bf16 in (False, True):
        with torch.no_grad(), _autocast(bf16):
            for _ in range(warmup):
                m(x, *args)
            torch.cuda.synchronize()
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
            evs[0].record()
            for i in range(steps):
                m(x, *args)
                evs[i + 1].record()
            torch.cuda.synchronize()
            ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))
            HGTConv.event_sink = []
            stages = {}
            for _ in range(steps):
                m(x, *args)
            torch.cuda.synchronize()
            for name, a, b in HGTConv.event_sink:
                stages.setdefault(name, []).append(a.elapsed_time(b))
            HGTConv.event_sink = None
            outs[bf16] = m(x, *args)
        st = {k: sorted(v)[len(v) // 2] for k, v in stages.items()}
        nbytes = edge_bytes(E, n_dst, d, rte, 2 if bf16 else 4)
        line = {"round": rnd, "config": config, "bf16_tables": bf16, "gpu": card[0], "power_limit": card[1],
                "workload": "%s: N=%d, E=%d, d=%d, H=%d, rte=%s" % (cfg["label"], N, E, d, H, rte),
                "ms_per_forward": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1],
                "edge_ms": st.get("edge"), "proj_linear_ms": st.get("proj_linear"),
                "edge_bytes_gb": round(nbytes / 1e9, 3),
                "edge_gbps": round(nbytes / 1e9 / (st["edge"] / 1e3), 1) if st.get("edge") else None}
        if bf16:
            diff = (outs[True] - outs[False]).double()
            line["max_abs_vs_fp32"] = float(diff.abs().max())
            line["rel_fro_vs_fp32"] = float(diff.norm() / outs[False].double().norm())
        print(json.dumps(line), flush=True)
    del m, x, outs


def train_lines(scale, steps, warmup, rnd, dev, card):
    cfg = bench.CONFIGS["c4"]
    D, H, L = cfg["d"], cfg["heads"], cfg["layers"]
    g = bench.make_graph("c4", scale)
    N, E, T, R = g.num_nodes, g.num_edges, g.num_types, g.num_relations
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([HGTConv(D, D, T, R, H, 0.0, True, False) for _ in range(L)]).to(dev).train()
    for m in layers:
        m.keep_att = False
    x = torch.randn(N, D, generator=torch.Generator().manual_seed(0)).to(dev)
    w = torch.randn(N, D, generator=torch.Generator().manual_seed(1)).to(dev)
    nt, ei, et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)

    def step(bf16):
        layers.zero_grad(set_to_none=True)
        h = x
        with _autocast(bf16):
            for m in layers:
                h = m(h, nt, ei, et)
        (h * w).sum().backward()

    for bf16 in (False, True):
        for _ in range(warmup):
            step(bf16)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        evs[0].record()
        for i in range(steps):
            step(bf16)
            evs[i + 1].record()
        torch.cuda.synchronize()
        ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))
        print(json.dumps({"round": rnd, "config": "c4", "bf16_tables": bf16, "gpu": card[0], "power_limit": card[1],
                          "workload": "%s: N=%d, E=%d, d=%d, H=%d, %d layers" % (cfg["label"], N, E, D, H, L),
                          "ms_per_step": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1],
                          "max_memory_allocated_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}), flush=True)
    del layers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--configs", default="c2,c3,c5,c4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bf16_tables_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = _card(dev)
    for rnd in range(args.rounds):
        for config in args.configs.split(","):
            if config == "c4":
                train_lines(args.scale, args.steps, args.warmup, rnd, dev, card)
            else:
                forward_lines(config, args.scale, args.steps, args.warmup, rnd, dev, card)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
