"""Eager training step with and without trimming (GNN.forward(..., out_nodes=) on the seed papers) on device-sampled
subgraphs, plus a variance-reduced eval forward in both modes.

Workload: graphed_train_bench.py's — the MAG-schema graph of gpu_sampler_bench.make_graph, 32 device-sampled subgraphs of
128 paper seeds per epoch (ONE sample_subgraphs_cuda call), at depth x width 6x520 (ogbn-mag recipe) and 3x64, the
ogbn-mag GNN (128 -> 512, 4 HGT layers, 8 heads, RTE, dropout 0.2), a linear head with log-softmax + nll_loss, AdamW /
OneCycleLR and clip_grad_norm_ 1.0.  The full and the trimmed step alternate epoch by epoch on the same 32 batches, each
from its own copy of the model; an epoch is timed with a host clock ending in a device synchronise and with CUDA events.
The trimmed step builds its hop layout every step (one read-back), as a training loop that sees each batch once does; a
third variant, trimmed_layout_cached, finds every layout (and its per-layer tables) built, which separates what the layers
save from what the layout build costs.  trimmed_signature builds the layout every step too, but from a TrimSignature (the
epoch's per-(type, hop) maximum, one read-back per epoch), so nothing is read back in the step.  full_graphed and
trimmed_graphed replay the whole step (copy-in, plan, layout, forward, backward, clip, AdamW) from a CUDA graph
(graphed.GraphedTrainStep over the epoch's GraphSignature), the trimmed one with the signature's layout inside the graph.

Eval: 8 unions, each of 8 members around one set of 128 seeds (one sample_subgraphs_cuda call per union, a different seed
set per union) merged into one batch (merge_batches); a no-grad forward reading every member's seed rows: full forward +
row select vs out_nodes = the union's seed rows, each eager and replayed by graphed.GraphedForward, and the trimmed eager
forward with its layout read back or from a signature.  Every timing cycles through all 8 unions (16 forwards), and the
eval TrimSignature and GraphSignature are sized over all of them, so a union is padded to the per-class maximum of the
eight, as an eval loop would size its signature over the unions of its epoch; the padding rows are reported.

With --profile, one more process-local pass records one prebuilt trimmed step and one full step with torch.profiler and
prints the CUDA time per kernel name of each (top entries), for the attribution in DESIGN.md section 7.1.

One JSON line per setting: median (and min / max over epochs) ms per step and per eval forward in each mode, card name and power limit, the mean
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
from graphed_train_bench import BATCHES, Model, recipe, signature  # noqa: E402

VR_MEMBERS = 8
VR_UNIONS = 8


def loss_of(model, batch, trimmed, tsig=None):
    (nf, nt, tm, ei, et), y, rows = batch
    if trimmed:
        h = model.gnn(nf, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig)
    else:
        h = model.gnn(nf, nt, tm, ei, et)[rows]
    return F.nll_loss(F.log_softmax(model.head(h), -1), y), h


def run_steps(model, opt, sched, batches, trimmed, tsig=None):
    for batch in batches:
        loss, _ = loss_of(model, batch, trimmed, tsig)
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for g in opt.param_groups for p in g["params"]], 1.0, foreach=True)
        opt.step()
        if sched is not None:
            sched.step()


def graphed_step(model, opt, sig, paper, tsig, trimmed):
    """GraphedTrainStep of the recipe's step on the seed papers (the first 128 papers of every padded batch)."""
    from pyhgt_b200 import graphed
    r0 = int(sig.row0[paper])
    rows = torch.arange(r0, r0 + 128, device="cuda")

    def loss_fn(x, nt, tm, ei, et, tg):
        if trimmed:
            h = model.gnn(x, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig)
        else:
            h = model.gnn(x, nt, tm, ei, et)[rows]
        return F.nll_loss(F.log_softmax(model.head(h), -1), tg[paper][:128], ignore_index=-100)

    kw = dict(optimizer=opt, clip_norm=1.0) if opt is not None else dict(params=list(model.parameters()))
    return graphed.GraphedTrainStep(loss_fn, sig, "cuda", targets={paper: ((), torch.int64, -100)}, **kw)


def run_graphed(step, sched, batches, paper):
    for b, y, _ in batches:
        loss, = step(*b, targets={paper: y})
        if sched is not None:
            sched.step()
    return loss


def profile(m, opt, batches, T, R):
    """CUDA time per kernel of one full and one prebuilt trimmed step (torch.profiler), in ms, top entries."""
    from torch.profiler import ProfilerActivity, profile as prof
    from pyhgt_b200 import trim
    out = {}
    for name, trimmed in (("full", False), ("trimmed_prebuilt", True)):
        one = batches[:1]
        if trimmed:
            (nf, nt, tm, ei, et), _, s_ = one[0]
            trim.get_layout(nt, ei, et, tm, s_, T, R, 4)
        run_steps(m, opt, None, one, trimmed)                                   # warm, with the layout built
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            run_steps(m, opt, None, one, trimmed)
            torch.cuda.synchronize()
        rows = sorted(((e.key, e.device_time_total / 1e3, e.count) for e in p.key_averages()), key=lambda r: -r[1])
        out[name] = {"total_ms": round(sum(r[1] for r in rows), 3),
                     "top": [(k[:60], round(v, 3), c) for k, v, c in rows[:25]]}
    return out


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
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import pyhgt_b200
    from pyhgt_b200 import graphed, plan as P, sampler, trim
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
        paper = dg.slot["paper"]
        sig, _ = signature(dg, batches)
        tsig = trim.TrimSignature.for_batches([b for b, _, _ in batches], [s_ for _, _, s_ in batches], 4,
                                              num_types=T, num_relations=R)
        # rows of the layers' reach (hop classes 0..L) per batch, exact vs the signature's slots (+ the pad row)
        exact = [int(trim.get_layout(b[1], b[3], b[4], b[2], s_, T, R, 4).bounds[:, :5].sum()) for b, _, s_ in batches]
        pad_rows = {"exact_rows_mean": float(np.mean(exact)), "exact_rows_max": int(max(exact)),
                    "signature_rows": tsig.n_rows, "padding_rows_mean": round(tsig.n_rows - float(np.mean(exact)), 1),
                    "batch_nodes_mean": real["nodes"], "graph_signature_nodes": sig.n_nodes}

        # parity, dropout 0: outputs and losses of the seed rows on the first batches
        torch.manual_seed(0)
        m0 = Model(T, R, 0.0).to(dev).train()
        d_out = d_loss = d_out_sig = d_loss_sig = d_loss_graphed = 0.0
        for batch in batches[:4]:
            lf, hf = loss_of(m0, batch, False)
            lt, ht = loss_of(m0, batch, True)
            ls, hs = loss_of(m0, batch, True, tsig)
            d_out = max(d_out, float((hf - ht).detach().abs().max()))
            d_loss = max(d_loss, abs(float(lf) - float(lt)))
            d_out_sig = max(d_out_sig, float((hf - hs).detach().abs().max()))
            d_loss_sig = max(d_loss_sig, abs(float(lf) - float(ls)))
        del lf, hf, lt, ht, ls, hs                          # a live autograd graph would break the captures below
        g_full, g_trim = graphed_step(m0, None, sig, paper, None, False), graphed_step(m0, None, sig, paper, tsig, True)
        for b, y, _ in batches[:4]:
            lf, = g_full(*b, targets={paper: y})
            lt, = g_trim(*b, targets={paper: y})
            d_loss_graphed = max(d_loss_graphed, abs(float(lf) - float(lt)))
        del g_full, g_trim

        torch.manual_seed(0)
        base = Model(T, R, 0.2).to(dev).train()
        total = (args.epochs + 1) * BATCHES + 1
        m_f, m_t = copy.deepcopy(base), copy.deepcopy(base)
        opt_f, sched_f = recipe(m_f, total)
        opt_t, sched_t = recipe(m_t, total)
        m_c = copy.deepcopy(base)
        opt_c, sched_c = recipe(m_c, total)
        m_s, m_fg, m_tg = copy.deepcopy(base), copy.deepcopy(base), copy.deepcopy(base)
        opt_s, sched_s = recipe(m_s, total)
        opt_fg, sched_fg = recipe(m_fg, total)
        opt_tg, sched_tg = recipe(m_tg, total)
        step_fg = graphed_step(m_fg, opt_fg, sig, paper, None, False)
        step_tg = graphed_step(m_tg, opt_tg, sig, paper, tsig, True)
        runs = {"full": lambda: run_steps(m_f, opt_f, sched_f, batches, False),
                "full_graphed": lambda: run_graphed(step_fg, sched_fg, batches, paper),
                "trimmed": lambda: run_steps(m_t, opt_t, sched_t, batches, True),
                "trimmed_layout_cached": lambda: run_steps(m_c, opt_c, sched_c, batches, True),
                "trimmed_signature": lambda: run_steps(m_s, opt_s, sched_s, batches, True, tsig),
                "trimmed_graphed": lambda: run_graphed(step_tg, sched_tg, batches, paper)}

        def prebuild(k):
            # "trimmed" builds every layout inside the step; "trimmed_layout_cached" finds them built (untimed): the
            # difference is what the layout build (BFS, reorder, read-back, hop plan, per-layer tiles) costs per step
            if k in ("trimmed", "trimmed_signature"):
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

        # variance-reduced eval: VR_UNIONS unions, each of 8 members around one seed set (a different set per union);
        # every timing cycles through all of them, so each forward sees another union, and the eval signature is sized
        # over all of them, as an eval loop would size it over its epoch
        unions = []
        for u in range(VR_UNIONS):
            members, _ = sample(dg, time_range, depth, width, year, paper_label, VR_MEMBERS, 1 + u, same_seeds=True)
            nf, nt, tm, ei, et, mrows = sampler.merge_batches([m[:5] for m in members], T, R)
            p0s = [P.get_plan(m[1], m[3], m[4], m[2], T, R).type_row0[paper] for m in members]
            unions.append(((nf, nt, tm, ei, et), torch.cat([r[p0:p0 + 128] for r, p0 in zip(mrows, p0s)])))
        del members
        m_e = copy.deepcopy(base).eval()
        n_eval = 2 * VR_UNIONS
        usig, _ = signature(dg, [(b, None, None) for b, _ in unions])
        esig = trim.TrimSignature.for_batches([b for b, _ in unions], [s_ for _, s_ in unions], 4, num_types=T,
                                              num_relations=R)
        # the seeds' rows in the padded static batch (papers of a union start at usig.row0[paper] there)
        static_rows = [s_ + (int(usig.row0[paper]) - P.get_plan(b[1], b[3], b[4], b[2], T, R).type_row0[paper])
                       for b, s_ in unions]
        rows_buf = static_rows[0].clone()                      # the graph's out_nodes, refilled before every replay
        ev_exact = [int(trim.get_layout(b[1], b[3], b[4], b[2], s_, T, R, 4).bounds[:, :5].sum()) for b, s_ in unions]
        ev_rows = {"unions": VR_UNIONS, "exact_rows_mean": float(np.mean(ev_exact)), "exact_rows_max": int(max(ev_exact)),
                   "signature_rows": esig.n_rows, "padding_rows_mean": round(esig.n_rows - float(np.mean(ev_exact)), 1),
                   "union_nodes_mean": float(np.mean([b[1].numel() for b, _ in unions])),
                   "graph_signature_nodes": usig.n_nodes}
        gf_full = graphed.GraphedForward(lambda x, a, b, c, d: m_e.gnn(x, a, b, c, d), usig, "cuda")
        gf_trim = graphed.GraphedForward(lambda x, a, b, c, d: m_e.gnn(x, a, b, c, d, out_nodes=rows_buf,
                                                                       trim_signature=esig),
                                         usig, "cuda", per_node=False)

        def ev_full():
            with torch.no_grad():
                for i in range(n_eval):
                    b, s_ = unions[i % VR_UNIONS]
                    m_e.gnn(*b)[s_]

        def ev_trim():
            with torch.no_grad():
                for i in range(n_eval):
                    b, s_ = unions[i % VR_UNIONS]
                    trim.clear_trim_cache()                                    # a new eval batch each time
                    m_e.gnn(*b, out_nodes=s_)

        def ev_sig():
            with torch.no_grad():
                for i in range(n_eval):
                    b, s_ = unions[i % VR_UNIONS]
                    trim.clear_trim_cache()
                    m_e.gnn(*b, out_nodes=s_, trim_signature=esig)

        def ev_graphed_full():
            for i in range(n_eval):
                b, s_ = unions[i % VR_UNIONS]
                gf_full(*b)[s_]

        def ev_graphed_trim():
            for i in range(n_eval):
                b, _ = unions[i % VR_UNIONS]
                rows_buf.copy_(static_rows[i % VR_UNIONS])
                gf_trim(*b)

        ev = {"full": ev_full, "full_graphed": ev_graphed_full, "trimmed": ev_trim, "trimmed_signature": ev_sig,
              "trimmed_graphed": ev_graphed_trim}
        for fn in ev.values():
            timed(fn, n_eval)
        ev_res = {k: [] for k in ev}
        for _ in range(args.epochs):
            for k, fn in ev.items():
                ev_res[k].append(timed(fn, n_eval))
        d_eval = {k: 0.0 for k in ("trimmed", "trimmed_signature", "full_graphed", "trimmed_graphed")}
        with torch.no_grad():
            for u, (b, s_) in enumerate(unions):
                ref = m_e.gnn(*b)[s_]
                rows_buf.copy_(static_rows[u])
                got = {"trimmed": m_e.gnn(*b, out_nodes=s_),
                       "trimmed_signature": m_e.gnn(*b, out_nodes=s_, trim_signature=esig),
                       "full_graphed": gf_full(*b)[s_], "trimmed_graphed": gf_trim(*b)}
                for k, v in got.items():
                    d_eval[k] = max(d_eval[k], float((ref - v).abs().max()))
        nt, ei = unions[0][0][1], unions[0][0][3]
        del gf_full, gf_trim, step_fg, step_tg
        prof = profile(m_c, opt_c, batches, T, R) if args.profile else None

        def med(v):
            return {"host_ms": round(float(np.median([h for h, _ in v])), 3),
                    "event_ms": round(float(np.median([e for _, e in v])), 3),
                    "event_ms_min_max": [round(float(min(e for _, e in v)), 3), round(float(max(e for _, e in v)), 3)]}

        step = {k: med(v) for k, v in res.items()}
        trim.clear_trim_cache()
        evm = {k: med(v) for k, v in ev_res.items()}
        print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128, "batches_per_epoch": BATCHES},
                          "graph": {"nodes": n, "edges": n_edges}, "epochs": args.epochs, "real_mean": real,
                          "train_step_ms": step,
                          "train_speedup_host": round(step["full"]["host_ms"] / step["trimmed"]["host_ms"], 3),
                          "vr_eval_forward_ms": evm,
                          "vr_eval": {"members": VR_MEMBERS, "unions": VR_UNIONS, "nodes_first": int(nt.numel()),
                                      "edges_first": int(ei.shape[1])},
                          "vr_eval_speedup_host": round(evm["full"]["host_ms"] / evm["trimmed"]["host_ms"], 3),
                          "layer_row_fraction": rows_frac, "layer_edge_fraction": edge_frac,
                          "max_abs_diff": {"out": d_out, "loss": d_loss, "out_signature": d_out_sig,
                                           "loss_signature": d_loss_sig, "loss_graphed": d_loss_graphed,
                                           "vr_eval_out": d_eval},
                          "hop_bound_rows": pad_rows, "vr_eval_hop_bound_rows": ev_rows, "profile": prof,
                          "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
