"""Sampling the next batch beside the current step: GraphedTrainStep.run / GraphedForward.run against step() loops.

Workload: the MAG-schema graph of gpu_sampler_bench.make_graph, 128 seed papers per subgraph, at each --settings
depth x width, and the ogbn-mag recipe model of graphed_train_bench.py (GNN 128 -> 512, 4 HGT layers, 8 heads, RTE,
dropout 0.2, linear head, AdamW capturable, clip 1.0).  Training variants, alternated round after round in one process:
  step      32 GraphedTrainStep(sampler=).step(seeds) calls: each replays the sampler's graph, then the step's;
  run       GraphedTrainStep.run(32 seed dicts): batch k + 1 sampled on the prefetch stream (priority
            sampler.PREFETCH_PRIORITY) while step k runs;
  run_p0    the same with the prefetch stream at the default priority 0;
  floor     the step alone on 32 pre-sampled batches (publish copies + the training graph, no sampling);
  sample    the 32 samples alone (the sampler's captured run on the prefetch stream, no training).
Variance-reduced forward (members=8), per forward of 8 subgraphs:
  vr_step   GraphedForward(sampler=).step(seeds) calls;
  vr_run    GraphedForward.run(seed dicts, consume) with a consume that keeps nothing;
  vr_floor  the forward alone on pre-sampled batches.
Reports CUDA-event ms per step, median and min-max over the rounds, with the card name and power limit read in the same
run; one JSON line per setting.  --profile instead runs one torch.profiler pass of `run` per setting, writes its trace
under --out, and reports the sampler-stream kernel time, the training-stream kernel time and how much of the first
overlaps the second.

    python scripts/prefetch_sampler_bench.py [--scale 0.5] [--rounds 3] [--settings 6x520,3x64] [--state-room 1e9]
                                             [--profile --out DIR]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_sampler_bench import F_IN, card, make_graph  # noqa: E402
from graphed_train_bench import Model, recipe  # noqa: E402

STEPS = 32
VR_STEPS = 16
SEEDS = 128
VR = 8


def _merge(intervals):
    out = []
    for a, b in sorted(intervals):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def _overlap(x, y):
    """Total length of the intersection of two merged interval lists."""
    i = j = 0
    tot = 0.0
    while i < len(x) and j < len(y):
        lo, hi = max(x[i][0], y[j][0]), min(x[i][1], y[j][1])
        tot += max(0.0, hi - lo)
        if x[i][1] < y[j][1]:
            i += 1
        else:
            j += 1
    return tot


def trace_overlap(path):
    """Kernel events of a chrome trace grouped by CUDA stream: the sampler stream is the one whose kernels include the
    hashed-state ones (k_hash*, k_hsel*); the training stream the other stream with the most kernel time."""
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    by_stream = {}
    for e in ev:
        if e.get("cat") == "kernel" and "dur" in e:
            by_stream.setdefault(e["args"].get("stream"), []).append((e["name"], float(e["ts"]), float(e["dur"])))
    samp = max(by_stream, key=lambda s: sum(("k_hash" in n or "k_hsel" in n) for n, _, _ in by_stream[s]))
    rest = [s for s in by_stream if s != samp]
    train = max(rest, key=lambda s: sum(d for _, _, d in by_stream[s]))
    iv = {s: _merge([(t, t + d) for _, t, d in by_stream[s]]) for s in (samp, train)}
    busy = {s: sum(b - a for a, b in iv[s]) for s in iv}
    both = _overlap(iv[samp], iv[train])
    return {"sampler_stream_busy_us": round(busy[samp], 1), "train_stream_busy_us": round(busy[train], 1),
            "overlap_us": round(both, 1), "sampler_time_overlapped": round(both / max(busy[samp], 1e-9), 3),
            "sampler_kernels": len(by_stream[samp]), "train_kernels": len(by_stream[train])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--settings", default="6x520,3x64")
    ap.add_argument("--state-room", type=float, default=1e9,
                    help="GraphedSampler state_room; 1e9 gives every region twice its id range (never overflows)")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the --profile trace (default: a new temporary one)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import pyhgt_b200
    import torch.nn.functional as F
    from pyhgt_b200 import graphed, sampler
    dev = torch.device("cuda:0")
    pyhgt_b200.HGTConv.keep_att = False
    g, n, year, _ = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    T, R = len(dg.types), len(dg.edge_dict)
    paper = dg.slot["paper"]
    time_range = {y: True for y in range(1990, 2016)}
    label = torch.from_numpy(rng.randint(0, 349, n["paper"])).to(dev)
    pool = np.nonzero(year <= 2015)[0]
    name, power = card()

    def inputs(seed, k):
        r = np.random.RandomState(seed)
        return [{"paper": np.stack([p, year[p]], 1)} for p in (r.choice(pool, SEEDS, replace=False) for _ in range(k))]

    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        probes = inputs(99, 16)
        sig1 = sampler.graph_signature_for(dg, depth, width, probes, 0.5, time_range=time_range)
        sig8 = sampler.graph_signature_for(dg, depth, width, probes, 0.5, members=VR, time_range=time_range)
        mk = lambda sig, B: sampler.GraphedSampler(dg, sig, depth, width, {"paper": SEEDS}, members=B,
                                                   time_range=time_range, state_room=args.state_room)
        gss = {"step": mk(sig1, 1), "run": mk(sig1, 1)}
        torch.manual_seed(0)
        steps = {}
        for v, gs in gss.items():
            m = Model(T, R, 0.2).to(dev)
            opt, _ = recipe(m, 10 ** 6)

            def loss(x, nt, tm, ei, et, tg, m=m, gs=gs):
                ids = gs.node_id
                y = torch.where((ids >= 0) & (nt == paper), label[ids.clamp(min=0)], torch.full_like(ids, -100))
                return F.nll_loss(F.log_softmax(m.head(m.gnn(x, nt, tm, ei, et)), -1), y, ignore_index=-100)
            steps[v] = graphed.GraphedTrainStep(loss, sig1, dev, optimizer=opt, clip_norm=1.0, sampler=gs)
        gs8 = mk(sig8, VR)
        evalm = Model(T, R, 0.0).to(dev).eval()
        fwd = graphed.GraphedForward(lambda x, nt, tm, ei, et: evalm.gnn(x, nt, tm, ei, et), sig8, dev, sampler=gs8)
        gsr = gss["run"]
        hi, lo = gsr.prefetch_stream, torch.cuda.Stream(device=dev, priority=0)

        def presample(gs, inps):
            out = []
            for inp in inps:
                gs.fill(inp)
                out.append([getattr(gs, k).clone() for k in ("x", "ei", "et", "tm", "node_id", "node_time")])
            return out

        def floor(obj, batches, replay):
            gs = obj.sampler
            cur = torch.cuda.current_stream()
            obj.stream.wait_stream(cur)
            with torch.cuda.stream(obj.stream):
                for b in batches:
                    for k, t in zip(("x", "ei", "et", "tm", "node_id", "node_time"), b):
                        getattr(gs, k).copy_(t)
                    replay()
            cur.wait_stream(obj.stream)

        def run_with(stream):
            def f(inps, _):
                gsr.prefetch_stream = stream
                steps["run"].run(inps)
                gsr.prefetch_stream = hi
            return f

        def sample_only(inps, _):
            staged = gsr.stage_batches(inps)
            for k in range(staged.n):
                gsr.sample_staged(staged, k)
            torch.cuda.current_stream().wait_stream(gsr.prefetch_stream)

        train = {
            "step": lambda inps, _: [steps["step"].step(i) for i in inps],
            "run": run_with(hi),
            "run_p0": run_with(lo),
            "floor": lambda _, pre: floor(steps["run"], pre, steps["run"].graph.replay),
            "sample": sample_only,
        }
        vr = {
            "vr_step": lambda inps, _: [fwd.step(i) for i in inps],
            "vr_run": lambda inps, _: fwd.run(inps, lambda rows, ids: None),
            "vr_floor": lambda _, pre: floor(fwd, pre, fwd.graph.replay),
        }
        steps["step"].step(inputs(1, 1)[0])                # first calls: warm-up + capture
        steps["run"].run(inputs(1, 2))
        fwd.step(inputs(1, 1)[0])
        fwd.run(inputs(1, 2), lambda rows, ids: None)
        torch.cuda.synchronize()

        if args.profile:
            if args.out is None:
                args.out = tempfile.mkdtemp(prefix="prefetch_trace_")
            os.makedirs(args.out, exist_ok=True)
            path = os.path.join(args.out, "prefetch_%s.pt.trace.json" % setting)
            inps = inputs(7, STEPS)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                steps["run"].run(inps)
                torch.cuda.synchronize()
            prof.export_chrome_trace(path)
            res = trace_overlap(path)
            res.update({"setting": setting, "card": name, "power_limit": power, "steps": STEPS, "trace": path})
            print(json.dumps(res), flush=True)
            continue

        times = {v: [] for v in list(train) + list(vr)}
        for rd in range(args.rounds):
            inps = inputs(100 + rd, STEPS)
            pre1 = presample(gss["step"], inps)
            vinps = inps[:VR_STEPS]
            pre8 = presample(gs8, vinps)
            torch.cuda.synchronize()
            for group, per, xs, pre in ((train, STEPS, inps, pre1), (vr, VR_STEPS, vinps, pre8)):
                for v, f in group.items():
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    f(xs, pre)
                    e1.record()
                    torch.cuda.synchronize()
                    times[v].append(e0.elapsed_time(e1) / per)
            del pre1, pre8
        fits = []
        for gs in (gss["step"], gsr, gs8):
            try:
                gs.check()
                fits.append("ok")
            except (ValueError, IndexError, KeyError) as e:
                fits.append(str(e))
        print(json.dumps({
            "setting": setting, "card": name, "power_limit": power, "scale": args.scale, "rounds": args.rounds,
            "steps_per_round": STEPS, "vr_forwards_per_round": VR_STEPS, "vr_members": VR,
            "prefetch_priority": sampler.PREFETCH_PRIORITY,
            "ms_per_step": {v: {"median": round(float(np.median(t)), 3), "min": round(min(t), 3), "max": round(max(t), 3)}
                            for v, t in times.items()},
            "signature_b1": {"rows": sig1.n_nodes, "edges": sig1.n_edges},
            "signature_b8": {"rows": sig8.n_nodes, "edges": sig8.n_edges},
            "last_check": fits,
        }), flush=True)


if __name__ == "__main__":
    main()
