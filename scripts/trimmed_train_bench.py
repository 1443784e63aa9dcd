"""Eager training step with and without trimming (GNN.forward(..., out_nodes=) on the seed papers) on device-sampled
subgraphs, plus a variance-reduced eval forward in both modes.

Workload: graphed_train_bench.py's — the MAG-schema graph of gpu_sampler_bench.make_graph, 32 device-sampled subgraphs of
128 paper seeds per epoch (ONE sample_subgraphs_cuda call), at depth x width 6x520 (ogbn-mag recipe) and 3x64, the
ogbn-mag GNN (128 -> 512, 4 HGT layers, 8 heads, RTE, dropout 0.2), a linear head with log-softmax + nll_loss, AdamW /
OneCycleLR and clip_grad_norm_ 1.0.  The full and the trimmed step alternate epoch by epoch on the same 32 batches, each
from its own copy of the model; an epoch is timed with a host clock ending in a device synchronise and with CUDA events.
The trimmed step builds its hop layout every step (one read-back), as a training loop that sees each batch once does; a
third variant, trimmed_layout_cached, finds every layout (and its per-layer tables) built, which separates what the layers
save from what the layout build costs.

Eval: 8 members around the same 128 seeds (one sample_subgraphs_cuda call) merged into one batch (merge_batches), a
no-grad forward reading every member's seed rows: full forward + row select vs out_nodes = the union's seed rows.

One JSON line per setting: median ms per step and per eval forward in both modes, card name and power limit, the mean
per-layer fractions of destination rows and of their in-edges the trimmed layers compute, and, on the first batches with
dropout 0, the maximum difference of the seed rows' output and of the loss between the two modes.

    python scripts/trimmed_train_bench.py [--scale 1.0] [--epochs 5] [--settings 6x520,3x64]
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

from gpu_sampler_bench import card, make_graph  # noqa: E402
from graphed_train_bench import BATCHES, Model, recipe  # noqa: E402

VR_MEMBERS = 8


def loss_of(model, batch, trimmed):
    (nf, nt, tm, ei, et), y, rows = batch
    if trimmed:
        h = model.gnn(nf, nt, tm, ei, et, out_nodes=rows)
    else:
        h = model.gnn(nf, nt, tm, ei, et)[rows]
    return F.nll_loss(F.log_softmax(model.head(h), -1), y), h


def run_steps(model, opt, sched, batches, trimmed):
    for batch in batches:
        loss, _ = loss_of(model, batch, trimmed)
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for g in opt.param_groups for p in g["params"]], 1.0, foreach=True)
        opt.step()
        sched.step()


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n, e0.elapsed_time(e1) / n


def sample(dg, time_range, depth, width, year, paper_label, B, seed, same_seeds=False):
    from pyhgt_b200 import plan as P, sampler
    rng = np.random.RandomState(seed)
    pool = np.nonzero(year <= 2015)[0]
    inps = []
    p = rng.choice(pool, 128, replace=False)
    for _ in range(B):
        if not same_seeds:
            p = rng.choice(pool, 128, replace=False)
        inps.append({"paper": np.stack([p, year[p]], 1)})
    members = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(seed))
    out = []
    for m, inp in zip(members, inps):
        y = torch.from_numpy(paper_label[inp["paper"][:, 0]]).to(dg.device)
        p0 = P.get_plan(m[1], m[3], m[4], m[2], len(dg.types), len(dg.edge_dict)).type_row0[dg.slot["paper"]]
        out.append((m[:5], y, torch.arange(p0, p0 + 128, device=dg.device)))    # seeds are the first papers
    return members, out


def fractions(batches, T, R, L):
    """Mean over batches of the share of destination rows (and of their in-edges) each trimmed layer computes."""
    from pyhgt_b200 import trim
    rows, edges = np.zeros(L), np.zeros(L)
    for (nf, nt, tm, ei, et), _, s in batches:
        lay = trim.get_layout(nt, ei, et, tm, s, T, R, L)
        rp = lay.plan.row_ptr.cpu().numpy()
        N, E = lay.plan.n_nodes, max(lay.plan.n_edges, 1)
        for l, v in enumerate(lay.layers):
            rows[l] += sum(v.active) / N
            edges[l] += sum(int(rp[lay.plan.type_row0[t] + a] - rp[lay.plan.type_row0[t]])
                            for t, a in enumerate(v.active)) / E
    return [round(v / len(batches), 3) for v in rows], [round(v / len(batches), 3) for v in edges]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--settings", default="6x520,3x64")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import pyhgt_b200
    from pyhgt_b200 import plan as P, sampler, trim
    dev = torch.device("cuda:0")
    P._CACHE_SIZE = 2 * BATCHES + 8                      # the epoch's plans stay cached for the full step (as graphed_train_bench)
    trim._CACHE_SIZE = BATCHES + 8                       # room for an epoch of prebuilt layouts (trimmed_layout_cached)
    pyhgt_b200.HGTConv.keep_att = False
    g, n, year, n_edges = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), 128).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    paper_label = rng.randint(0, 349, n["paper"]).astype(np.int64)
    time_range = {y: True for y in range(1990, 2016)}
    T, R = len(dg.types), len(dg.edge_dict)
    name, power = card()
    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        _, batches = sample(dg, time_range, depth, width, year, paper_label, BATCHES, 0)
        real = {"nodes": float(np.mean([b[0][1].numel() for b in batches])),
                "edges": float(np.mean([b[0][3].shape[1] for b in batches]))}
        rows_frac, edge_frac = fractions(batches, T, R, 4)

        # parity, dropout 0: outputs and losses of the seed rows on the first batches
        torch.manual_seed(0)
        m0 = Model(T, R, 0.0).to(dev).train()
        d_out = d_loss = 0.0
        for batch in batches[:4]:
            lf, hf = loss_of(m0, batch, False)
            lt, ht = loss_of(m0, batch, True)
            d_out = max(d_out, float((hf - ht).detach().abs().max()))
            d_loss = max(d_loss, abs(float(lf) - float(lt)))

        torch.manual_seed(0)
        base = Model(T, R, 0.2).to(dev).train()
        total = (args.epochs + 1) * BATCHES + 1
        m_f, m_t = copy.deepcopy(base), copy.deepcopy(base)
        opt_f, sched_f = recipe(m_f, total)
        opt_t, sched_t = recipe(m_t, total)
        m_c = copy.deepcopy(base)
        opt_c, sched_c = recipe(m_c, total)
        runs = {"full": lambda: run_steps(m_f, opt_f, sched_f, batches, False),
                "trimmed": lambda: run_steps(m_t, opt_t, sched_t, batches, True),
                "trimmed_layout_cached": lambda: run_steps(m_c, opt_c, sched_c, batches, True)}

        def prebuild(k):
            # "trimmed" builds every layout inside the step; "trimmed_layout_cached" finds them built (untimed): the
            # difference is what the layout build (BFS, reorder, read-back, hop plan, per-layer tiles) costs per step
            if k == "trimmed":
                trim.clear_trim_cache()
            if k == "trimmed_layout_cached":
                for (nf, nt, tm, ei, et), _, s_ in batches:
                    trim.get_layout(nt, ei, et, tm, s_, T, R, 4)

        for k, fn in runs.items():                                             # warm-up epoch of each
            prebuild(k)
            timed(fn, BATCHES)
        res = {k: [] for k in runs}
        for _ in range(args.epochs):
            for k, fn in runs.items():
                prebuild(k)
                res[k].append(timed(fn, BATCHES))

        # variance-reduced eval: 8 members around the same seeds, one union batch
        members, _ = sample(dg, time_range, depth, width, year, paper_label, VR_MEMBERS, 1, same_seeds=True)
        nf, nt, tm, ei, et, mrows = sampler.merge_batches([m[:5] for m in members], T, R)
        p0s = [P.get_plan(m[1], m[3], m[4], m[2], T, R).type_row0[dg.slot["paper"]] for m in members]
        s = torch.cat([r[p0:p0 + 128] for r, p0 in zip(mrows, p0s)])
        m_e = copy.deepcopy(base).eval()
        n_eval = 10

        def ev_full():
            with torch.no_grad():
                for _ in range(n_eval):
                    m_e.gnn(nf, nt, tm, ei, et)[s]

        def ev_trim():
            from pyhgt_b200 import trim
            with torch.no_grad():
                for _ in range(n_eval):
                    trim.clear_trim_cache()                                    # a new eval batch each time
                    m_e.gnn(nf, nt, tm, ei, et, out_nodes=s)

        ev = {"full": ev_full, "trimmed": ev_trim}
        for fn in ev.values():
            timed(fn, n_eval)
        ev_res = {k: [] for k in ev}
        for _ in range(args.epochs):
            for k, fn in ev.items():
                ev_res[k].append(timed(fn, n_eval))
        with torch.no_grad():
            d_eval = float((m_e.gnn(nf, nt, tm, ei, et)[s] - m_e.gnn(nf, nt, tm, ei, et, out_nodes=s)).abs().max())

        def med(v):
            return {"host_ms": round(float(np.median([h for h, _ in v])), 3),
                    "event_ms": round(float(np.median([e for _, e in v])), 3)}

        step = {k: med(v) for k, v in res.items()}
        trim.clear_trim_cache()
        evm = {k: med(v) for k, v in ev_res.items()}
        print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128, "batches_per_epoch": BATCHES},
                          "graph": {"nodes": n, "edges": n_edges}, "epochs": args.epochs, "real_mean": real,
                          "train_step_ms": step,
                          "train_speedup_host": round(step["full"]["host_ms"] / step["trimmed"]["host_ms"], 3),
                          "vr_eval_forward_ms": evm,
                          "vr_eval": {"members": VR_MEMBERS, "nodes": int(nt.numel()), "edges": int(ei.shape[1])},
                          "vr_eval_speedup_host": round(evm["full"]["host_ms"] / evm["trimmed"]["host_ms"], 3),
                          "layer_row_fraction": rows_frac, "layer_edge_fraction": edge_frac,
                          "max_abs_diff": {"out": d_out, "loss": d_loss, "vr_eval_out": d_eval},
                          "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
