"""Eager vs CUDA-graph-replayed training step (graphed.GraphedTrainStep) on device-sampled subgraphs.

Workload: the MAG-schema graph of gpu_sampler_bench.make_graph (2.3 M edges at --scale 1, counting the rev_* twins and
'self' loops), 128 paper seeds per
subgraph, at the ogbn-mag recipe setting (depth 6, width 520; pyHGT ogbn-mag/train_ogbn_mag.py:44-47) and a small one
(depth 3, width 64).  An epoch is the 32 subgraphs of ONE sample_subgraphs_cuda call.  Model and recipe are ogbn-mag's
(train_ogbn_mag.py:108-129, 170-178): GNN(128 -> 512, 4 HGT layers, 8 heads, RTE, dropout 0.2) and a linear head with
log-softmax + nll_loss (labels on the seed papers, -100 elsewhere), AdamW (capturable, tensor lr, weight decay 0.01 /
0 groups, eps 1e-6), OneCycleLR (max_lr 5e-4, pct_start 0.05, linear, final_div_factor 10) and clip_grad_norm_ 1.0, with one change for
both paths: cycle_momentum=False, because a captured step holds AdamW's betas by value (the reference cycles beta1).
The graphed signature is the per-type maximum over the epoch's subgraphs; the plan cache is raised to hold the epoch's
plans (eager and graphed alike read them).

Eager and graphed epochs alternate (--epochs of each, same 32 subgraphs); each epoch is timed with a host clock that ends
in a device synchronise and with CUDA events.  One JSON line per setting: ms per step (median over epochs), the capture
time (first graphed call minus a replayed one), real vs padded nodes and edges, card name and power limit, and where
the eager-to-graphed difference goes, from three more variants timed in the same alternation: the eager step on the
padded batches (plan prebuilt: the padding's cost), the replay's work unrolled eagerly (copy-in + plan rebuild + step),
and the copy-in alone; plan rebuild = unrolled - eager_padded - copy_in, and unrolled - graphed is what the graph saves.
`--check`: one more line per setting with the eager and graphed losses on the same batches, dropout 0 and
torch.use_deterministic_algorithms on (max abs difference).
`--profile DIR`: instead of timing, torch.profiler traces of one eager step and one graphed replay per setting (written
under DIR), each with its GPU-busy fraction (union of device activity over the span from its first host op to its last
kernel) and top-kernel table.

    python scripts/graphed_train_bench.py [--scale 1.0] [--epochs 3] [--settings 6x520,3x64] [--check] [--profile DIR]
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_sampler_bench import F_IN, card, make_graph  # noqa: E402

N_CLS = 349
BATCHES = 32


class Model(torch.nn.Module):
    def __init__(self, T, R, dropout):
        super().__init__()
        from pyhgt_b200.model import GNN
        self.gnn = GNN(F_IN, 512, T, R, 8, 4, dropout, "hgt", True, True, True)
        self.head = torch.nn.Linear(512, N_CLS)

    def loss(self, x, nt, tm, ei, et, y, r0):
        h = self.gnn(x, nt, tm, ei, et)[r0:r0 + y.shape[0]]
        return F.nll_loss(F.log_softmax(self.head(h), -1), y, ignore_index=-100)


def recipe(model, total_steps):
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    opt = torch.optim.AdamW(groups, eps=1e-6, lr=torch.tensor(5e-4, device="cuda"), capturable=True)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, pct_start=0.05, anneal_strategy="linear", final_div_factor=10,
                                                max_lr=5e-4, total_steps=total_steps, cycle_momentum=False)
    return opt, sched


def epoch_batches(dg, time_range, depth, width, year, paper_label, epoch_seed):
    from pyhgt_b200 import plan as P, sampler
    rng = np.random.RandomState(epoch_seed)
    pool = np.nonzero(year <= 2015)[0]
    inps = []
    for _ in range(BATCHES):
        p = rng.choice(pool, 128, replace=False)
        inps.append({"paper": np.stack([p, year[p]], 1)})
    members = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(epoch_seed))
    out = []
    for m, inp in zip(members, inps):
        y = torch.from_numpy(paper_label[inp["paper"][:, 0]]).to(dg.device)       # seeds are the first papers
        p0 = P.get_plan(m[1], m[3], m[4], m[2], len(dg.types), len(dg.edge_dict)).type_row0[dg.slot["paper"]]
        out.append((m[:5], y, p0))
    return out


def signature(dg, batches):
    from pyhgt_b200 import graphed, plan as P
    T, R = len(dg.types), len(dg.edge_dict)
    plans = [P.get_plan(b[1], b[3], b[4], b[2], T, R) for b, _, _ in batches]
    counts = [max(p.type_count[t] for p in plans) for t in range(T)]
    pairs = {pr for p in plans for pr in p.pairs}
    sig = graphed.GraphSignature(counts, max(p.n_edges for p in plans), pairs, R, dg.feat_dim)
    real = {"nodes": float(np.mean([p.n_nodes for p in plans])), "edges": float(np.mean([p.n_edges for p in plans]))}
    return sig, real


def run_eager(model, opt, sched, batches, paper):
    for (nf, nt, tm, ei, et), y, p0 in batches:
        loss = model.loss(nf, nt, tm, ei, et, y, p0)
        opt.zero_grad()
        loss.backward()
        # the optimizer's parameter order, as GraphedTrainStep clips: the norm's sum order is part of the result
        torch.nn.utils.clip_grad_norm_([p for g in opt.param_groups for p in g["params"]], 1.0, foreach=True)
        opt.step()
        sched.step()
    return loss


def padded_batches(sig, batches, dev, T, R, paper):
    """Every member padded to the signature on the host, uploaded, with its sync-free plan built and cached: the eager step
    on exactly the graph's inputs, without the copy-in or the plan build."""
    from pyhgt_b200 import graphed, plan as P
    out = []
    for (nf, nt, tm, ei, et), y, _ in batches:
        padded = graphed.pad_batch(sig, nf.cpu(), nt.cpu(), tm.cpu(), ei.cpu(), et.cpu())[:5]
        tens = tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in padded)
        P.rebuild_plan(tens[1], tens[3], tens[4], tens[2], T, R, sig.host_meta())
        tgt = torch.full((sig.type_counts[paper],), -100, dtype=torch.int64, device=dev)
        tgt[:y.numel()] = y
        out.append((tens, tgt, int(sig.row0[paper])))
    return out


def run_unrolled(step, opt, sched, batches, paper, copy_only=False):
    """What one replay does, eagerly, through a GraphedTrainStep that is never captured: copy-in (hgt_merge_batches +
    fills) and target copy, then (unless copy_only) the plan rebuild, forward, backward, clip and update."""
    cur = torch.cuda.current_stream()
    for batch, y, _ in batches:
        step.stream.wait_stream(cur)
        with torch.cuda.stream(step.stream):
            step._feed(batch, step._sizes(batch))
            step._copy_targets({paper: y})
            if not copy_only:
                opt.zero_grad()
                step._step()
                sched.step()
        cur.wait_stream(step.stream)


def run_graphed(step, sched, batches, paper):
    for (nf, nt, tm, ei, et), y, _ in batches:
        loss, = step(nf, nt, tm, ei, et, targets={paper: y})
        sched.step()
    return loss


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / BATCHES, e0.elapsed_time(e1) / BATCHES


def busy_fraction(prof, label):
    from torch.autograd import DeviceType
    dev_iv, host0 = [], None
    for e in prof.events():
        if e.name == label and e.device_type == DeviceType.CPU:
            host0 = e.time_range.start
        elif e.device_type == DeviceType.CUDA:
            dev_iv.append((e.time_range.start, e.time_range.end))
    dev_iv.sort()
    busy, cur_s, cur_e = 0.0, None, None
    for s, e in dev_iv:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        busy += cur_e - cur_s
    span = max(e for _, e in dev_iv) - host0
    return busy / span, span / 1e3, busy / 1e3, len(dev_iv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--settings", default="6x520,3x64")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import pyhgt_b200
    from pyhgt_b200 import graphed, plan as P, sampler
    dev = torch.device("cuda:0")
    # the plan cache holds the whole epoch: the samplers build every member's plan, and both the eager layers and the
    # graphed device feed read it (the default 8 entries would rebuild 24 of 32 plans with a read-back each)
    P._CACHE_SIZE = 2 * BATCHES + 8
    pyhgt_b200.HGTConv.keep_att = False
    g, n, year, n_edges = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    paper_label = rng.randint(0, N_CLS, n["paper"]).astype(np.int64)
    time_range = {y: True for y in range(1990, 2016)}
    T, R = len(dg.types), len(dg.edge_dict)
    paper = dg.slot["paper"]
    name, power = card()
    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        batches = epoch_batches(dg, time_range, depth, width, year, paper_label, 0)
        sig, real = signature(dg, batches)
        r0 = int(sig.row0[paper])
        pad = {"nodes": sig.n_nodes, "edges": sig.n_edges}
        torch.manual_seed(0)
        base = Model(T, R, 0.0 if args.check else 0.2).to(dev).train()

        if args.profile:
            model, m_g = copy.deepcopy(base), copy.deepcopy(base)
            opt, sched = recipe(model, 10 * BATCHES)
            opt_g, sched_g = recipe(m_g, 10 * BATCHES)
            step = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg: m_g.loss(x, nt, tm, ei, et, tg[paper], r0),
                                            sig, dev, optimizer=opt_g, clip_norm=1.0,
                                            targets={paper: ((), torch.int64, -100)})
            run_eager(model, opt, sched, batches[:4], paper)                      # warm-up
            run_graphed(step, sched_g, batches[:4], paper)                        # warm-up + capture
            torch.cuda.synchronize()
            acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
            os.makedirs(args.profile, exist_ok=True)
            for label, fn in (("eager_step", lambda: run_eager(model, opt, sched, batches[4:5], paper)),
                              ("graphed_step", lambda: run_graphed(step, sched_g, batches[4:5], paper))):
                with torch.profiler.profile(activities=acts) as prof:
                    with torch.profiler.record_function(label):
                        fn()
                    torch.cuda.synchronize()
                stem = os.path.join(args.profile, "%s_%dx%d" % (label, depth, width))
                prof.export_chrome_trace(stem + ".pt.trace.json")
                frac, span_ms, busy_ms, n_act = busy_fraction(prof, label)
                with open(stem + ".txt", "w") as f:
                    f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
                print(json.dumps({"setting": setting, "profile": label, "gpu_busy_fraction": round(frac, 3),
                                  "span_ms": round(span_ms, 3), "device_busy_ms": round(busy_ms, 3),
                                  "device_activities": n_act, "gpu": name, "power_limit": power}), flush=True)
            continue

        if args.check:
            torch.use_deterministic_algorithms(True, warn_only=True)
            m_e, m_g = copy.deepcopy(base), copy.deepcopy(base)
            opt_e, sched_e = recipe(m_e, 10 * BATCHES)
            opt_g, sched_g = recipe(m_g, 10 * BATCHES)
            step = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg: m_g.loss(x, nt, tm, ei, et, tg[paper], r0),
                                            sig, dev, optimizer=opt_g, clip_norm=1.0,
                                            targets={paper: ((), torch.int64, -100)})
            le, lg = [], []
            for (nf, nt, tm, ei, et), y, p0 in batches[:8]:
                # eager on the same padded inputs and the same sync-free plan as the graph
                padded = graphed.pad_batch(sig, nf.cpu(), nt.cpu(), tm.cpu(), ei.cpu(), et.cpu())[:5]
                tens = tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in padded)
                P.rebuild_plan(tens[1], tens[3], tens[4], tens[2], T, R, sig.host_meta())
                tgt = torch.full((sig.type_counts[paper],), -100, dtype=torch.int64, device=dev)
                tgt[:y.numel()] = y
                le.append(run_eager(m_e, opt_e, sched_e, [(tens, tgt, r0)], paper).detach().clone())
                lg.append(run_graphed(step, sched_g, [((nf, nt, tm, ei, et), y, p0)], paper).clone())
            (nf, nt, tm, ei, et), y, p0 = batches[0]
            with torch.no_grad():
                first_unpadded = base.loss(nf, nt, tm, ei, et, y, p0).item()
            le, lg = torch.stack(le).cpu(), torch.stack(lg).cpu()
            torch.use_deterministic_algorithms(False)
            print(json.dumps({"setting": setting, "check": "eager on the padded batch vs graphed, dropout 0, deterministic",
                              "eager": le.tolist(), "graphed": lg.tolist(),
                              "max_abs_diff": float((le - lg).abs().max()),
                              "first_loss_unpadded_minus_graphed": first_unpadded - float(lg[0])}), flush=True)
            continue

        m_e, m_g = copy.deepcopy(base), copy.deepcopy(base)
        total = (args.epochs + 1) * BATCHES + 1
        opt_e, sched_e = recipe(m_e, total)
        opt_g, sched_g = recipe(m_g, total)
        step = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg: m_g.loss(x, nt, tm, ei, et, tg[paper], r0),
                                        sig, dev, optimizer=opt_g, clip_norm=1.0, targets={paper: ((), torch.int64, -100)})
        # warm-up epoch of each; the graphed one includes the capture, timed on its own
        timed(lambda: run_eager(m_e, opt_e, sched_e, batches, paper))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run_graphed(step, sched_g, batches[:1], paper)
        torch.cuda.synchronize()
        first_ms = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        run_graphed(step, sched_g, batches[1:2], paper)
        torch.cuda.synchronize()
        replay_ms = (time.perf_counter() - t0) * 1e3
        run_graphed(step, sched_g, batches[2:], paper)
        # where the difference goes: the eager step on the padded inputs (plan cached), the replay's work unrolled
        # eagerly (copy-in + in-graph plan rebuild + step), and the copy-in alone
        m_p, m_u = copy.deepcopy(base), copy.deepcopy(base)
        opt_p, sched_p = recipe(m_p, total)
        opt_u, sched_u = recipe(m_u, total)
        padded = padded_batches(sig, batches, dev, T, R, paper)
        unrolled = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg: m_u.loss(x, nt, tm, ei, et, tg[paper], r0),
                                            sig, dev, optimizer=opt_u, clip_norm=1.0,
                                            targets={paper: ((), torch.int64, -100)})
        timed(lambda: run_eager(m_p, opt_p, sched_p, padded, paper))
        timed(lambda: run_unrolled(unrolled, opt_u, sched_u, batches, paper))
        runs = {"eager": lambda: run_eager(m_e, opt_e, sched_e, batches, paper),
                "eager_padded": lambda: run_eager(m_p, opt_p, sched_p, padded, paper),
                "unrolled_replay": lambda: run_unrolled(unrolled, opt_u, sched_u, batches, paper),
                "copy_in_only": lambda: run_unrolled(unrolled, opt_u, sched_u, batches, paper, copy_only=True),
                "graphed": lambda: run_graphed(step, sched_g, batches, paper)}
        res = {k: [] for k in runs}
        for _ in range(args.epochs):
            for k, fn in runs.items():
                res[k].append(timed(fn))
        med = {k: {"host_ms_per_step": round(float(np.median([h for h, _ in v])), 3),
                   "event_ms_per_step": round(float(np.median([e for _, e in v])), 3),
                   "host_ms_per_epoch_step_all": [round(h, 3) for h, _ in v]} for k, v in res.items()}
        ev = {k: v["event_ms_per_step"] for k, v in med.items()}
        print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128, "batches_per_epoch": BATCHES},
                          "graph": {"nodes": n, "edges": n_edges}, "epochs": args.epochs,
                          "eager": med["eager"], "graphed": med["graphed"],
                          "breakdown_event_ms_per_step": {k: ev[k] for k in runs},
                          "attribution_ms": {"padding": round(ev["eager_padded"] - ev["eager"], 3),
                                             "copy_in": ev["copy_in_only"],
                                             "plan_rebuild": round(ev["unrolled_replay"] - ev["eager_padded"]
                                                                   - ev["copy_in_only"], 3),
                                             "removed_by_graph": round(ev["unrolled_replay"] - ev["graphed"], 3)},
                          "speedup_host": round(med["eager"]["host_ms_per_step"] / med["graphed"]["host_ms_per_step"], 3),
                          "capture_ms": round(first_ms - replay_ms, 1), "first_call_ms": round(first_ms, 1),
                          "real_mean": real, "padded": pad,
                          "padding_overhead": {"nodes": round(pad["nodes"] / real["nodes"], 3),
                                               "edges": round(pad["edges"] / real["edges"], 3)},
                          "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
