"""The captured sampler (sampler.GraphedSampler) feeding the captured training step against the eager sampler.

Workload: the MAG-schema graph of gpu_sampler_bench.make_graph, the ogbn-mag recipe model of graphed_train_bench.py
(GNN 128 -> 512, 4 HGT layers, 8 heads, RTE, dropout 0.2, linear head, AdamW capturable), 128 seed papers per subgraph,
at each --settings depth x width.  Variants, alternated round after round in one run:
  a  sample_subgraph_cuda per step, then a GraphedTrainStep replay fed that device batch;
  b  one sample_subgraphs_cuda(B=32) per 32 steps, then 32 GraphedTrainStep replays;
  c  32 GraphedTrainStep(sampler=GraphedSampler(...)).step calls: a sampler replay, then the step's (plan, step);
  d  eager sample_subgraphs_cuda(B=8) + merge_batches + forward (variance-reduced evaluation);
  e  GraphedForward(sampler=GraphedSampler(..., members=8)): the same as a sampler replay and a forward replay.
Per variant: ms per step from CUDA events and from a host clock ending in a synchronise, host CPU time per step, host
synchronisations per step (counted in an untimed pass with torch.cuda.set_sync_debug_mode("warn")), the padding of the
signature, the first call's time (warm-up + capture), and the card's name and power limit read in the same run.  One
JSON line per setting.

A run whose last fill overflowed its hashed regions or signature says so in "last_fill_check": its GraphedSampler
times are those of overflowing batches (long hash probes) and do not count.

    python scripts/graphed_sampler_bench.py [--scale 1.0] [--rounds 3] [--settings 6x520,3x64] [--state-room R]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_sampler_bench import F_IN, card, make_graph  # noqa: E402
from graphed_train_bench import N_CLS, Model, recipe  # noqa: E402

STEPS = 32
SEEDS = 128
VR = 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--settings", default="6x520,3x64")
    ap.add_argument("--state-room", type=float, default=None,
                    help="GraphedSampler state_room (default: the graph's); 1e9 gives every region twice its id range")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import pyhgt_b200
    import torch.nn.functional as F
    from pyhgt_b200 import graphed, plan as P, sampler
    dev = torch.device("cuda:0")
    P._CACHE_SIZE = 2 * STEPS + 8
    pyhgt_b200.HGTConv.keep_att = False
    g, n, year, _ = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    T, R = len(dg.types), len(dg.edge_dict)
    paper = dg.slot["paper"]
    time_range = {y: True for y in range(1990, 2016)}
    label = torch.from_numpy(rng.randint(0, N_CLS, n["paper"])).to(dev)
    pool = np.nonzero(year <= 2015)[0]
    name, power = card()

    def inputs(seed, k):
        r = np.random.RandomState(seed)
        out = []
        for _ in range(k):
            p = r.choice(pool, SEEDS, replace=False)
            out.append({"paper": np.stack([p, year[p]], 1)})
        return out

    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        probes = inputs(99, 16)
        sig1 = sampler.graph_signature_for(dg, depth, width, probes, 0.5, time_range=time_range)
        sig8 = sampler.graph_signature_for(dg, depth, width, probes, 0.5, members=VR, time_range=time_range)
        gs1 = sampler.GraphedSampler(dg, sig1, depth, width, {"paper": SEEDS}, time_range=time_range,
                                     state_room=args.state_room)
        gs8 = sampler.GraphedSampler(dg, sig8, depth, width, {"paper": SEEDS}, members=VR, time_range=time_range,
                                     state_room=args.state_room)
        torch.manual_seed(0)
        models = {v: Model(T, R, 0.2).to(dev) for v in "abc"}
        r0 = int(sig1.row0[paper])
        steps, opts = {}, {}
        for v in "ab":
            m = models[v]
            opts[v], _ = recipe(m, 10 ** 6)
            steps[v] = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg, m=m: m.loss(x, nt, tm, ei, et, tg[paper], r0),
                                                sig1, dev, optimizer=opts[v], clip_norm=1.0,
                                                targets={paper: ((), torch.int64, -100)})
        mc = models["c"]
        opts["c"], _ = recipe(mc, 10 ** 6)

        def loss_c(x, nt, tm, ei, et, tg):
            ids = gs1.node_id
            y = torch.where((ids >= 0) & (nt == paper), label[ids.clamp(min=0)], torch.full_like(ids, -100))
            return F.nll_loss(F.log_softmax(mc.head(mc.gnn(x, nt, tm, ei, et)), -1), y, ignore_index=-100)
        steps["c"] = graphed.GraphedTrainStep(loss_c, sig1, dev, optimizer=opts["c"], clip_norm=1.0, sampler=gs1)
        evalm = Model(T, R, 0.0).to(dev).eval()
        fn = lambda x, nt, tm, ei, et: evalm.gnn(x, nt, tm, ei, et)
        fwd = graphed.GraphedForward(fn, sig8, dev, sampler=gs8)
        gen = torch.Generator().manual_seed(0)

        def y_of(inp):
            return label[torch.from_numpy(inp["paper"][:, 0]).to(dev)]

        def run_a(inps):
            for inp in inps:
                b = sampler.sample_subgraph_cuda(dg, time_range, depth, width, inp, gen)
                steps["a"](*b[:5], targets={paper: y_of(inp)})

        def run_b(inps):
            for b, inp in zip(sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, gen), inps):
                steps["b"](*b[:5], targets={paper: y_of(inp)})

        def run_c(inps):
            for inp in inps:
                steps["c"].step(inp)

        def run_d(inps):
            with torch.no_grad():
                for inp in inps[:STEPS // VR]:
                    merged = sampler.merge_batches(sampler.sample_subgraphs_cuda(dg, time_range, depth, width,
                                                                                 [inp] * VR, gen), T, R)
                    fn(*merged[:5])

        def run_e(inps):
            for inp in inps[:STEPS // VR]:
                fwd.step(inp)

        runs = {"a": run_a, "b": run_b, "c": run_c, "d": run_d, "e": run_e}
        per_call = {"a": STEPS, "b": STEPS, "c": STEPS, "d": STEPS // VR, "e": STEPS // VR}
        first = {}
        for v, f in runs.items():                          # first calls: warm-up + capture
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f(inputs(1, 1 if v != "b" else STEPS)[:1] if v != "b" else inputs(1, STEPS))
            torch.cuda.synchronize()
            first[v] = (time.perf_counter() - t0) * 1e3
        syncs = {}
        for v, f in runs.items():
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("warn")
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                f(inputs(2, STEPS))
            torch.cuda.set_sync_debug_mode(0)
            syncs[v] = sum("synchroniz" in str(x.message) for x in w) / per_call[v]
        times = {v: [] for v in runs}
        for rd in range(args.rounds):
            for v, f in runs.items():
                inps = inputs(100 + rd, STEPS)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                c0, t0 = time.process_time(), time.perf_counter()
                e0.record()
                f(inps)
                e1.record()
                torch.cuda.synchronize()
                wall, cpu = time.perf_counter() - t0, time.process_time() - c0
                times[v].append((e0.elapsed_time(e1) / per_call[v], wall * 1e3 / per_call[v], cpu * 1e3 / per_call[v]))
        fits = []
        for gs in (gs1, gs8):
            try:
                gs.check()
                fits.append("ok")
            except (ValueError, IndexError, KeyError) as e:     # the last batch overflowed its signature
                fits.append(str(e))
        med = {v: [float(np.median([t[i] for t in times[v]])) for i in range(3)] for v in runs}
        real_rows = int((gs1.node_id >= 0).sum())
        print(json.dumps({
            "setting": setting, "card": name, "power_limit": power, "scale": args.scale, "rounds": args.rounds,
            "steps_per_round": STEPS, "vr_members": VR,
            "variants": {v: {"ms_per_step_events": round(med[v][0], 3), "ms_per_step_host": round(med[v][1], 3),
                             "host_cpu_ms_per_step": round(med[v][2], 3), "host_syncs_per_step": syncs[v],
                             "first_call_ms": round(first[v], 1), "unit": "step" if v in "abc" else "forward of %d" % VR}
                         for v in runs},
            "signature_b1": {"rows": sig1.n_nodes, "edges": sig1.n_edges, "last_real_rows": real_rows},
            "signature_b8": {"rows": sig8.n_nodes, "edges": sig8.n_edges},
            "last_fill_check": fits,
            "sampler_b1": {"sort_positions": gs1.n_sort, "region_entries_max": gs1.max_room},
        }), flush=True)


if __name__ == "__main__":
    main()
