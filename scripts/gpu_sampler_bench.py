"""Host HGSampling vs device HGSampling per batch, next to the training step they feed.

Workload: a seeded synthetic heterograph with the MAG schema (paper / author / field / venue, every relation with its
rev_* twin, 'self' loops on every type; about 1 M edges), frozen once (sampler.FrozenGraph) and uploaded once
(sampler.DeviceGraph).  Each setting samples from 128 paper seeds; the recipe setting is depth 6, width 520
(pyHGT ogbn-mag/train_ogbn_mag.py:44-47), the small one depth 3, width 64.

Prints one JSON line per setting:
  host_ms        sample_subgraph (batched native path, one process) + to_torch onto the device with the sync-free plan,
                 wall clock, median over --host-batches;
  device_ms      sample_subgraph_cuda (same outputs, features gathered on the device), CUDA events after warm-up,
                 median over --batches (>= 20);
  device_ms_per_subgraph
                 sample_subgraphs_cuda with B = 1, 8, 32 seed dicts per call, CUDA events / B, median;
  train_ms       fwd + bwd of a 4-layer n_hid=512 GNN (HGT) on one device batch, CUDA events, median;
  plus the batch sizes, the card name and its power limit.
Then one `edge_mask` line: `device_ms_per_subgraph` with the OAG paper-field label mask and without it, alternating
call by call, at every setting and B = 1, 8, 32.
Then one `vr_eval` line: 8 subgraphs of the first setting around the same 128 seeds, the GNN plus a linear head under
eval() / no_grad, timed as 8 single samples + 8 forwards and as one batched sample + merge_batches + one forward, with
the max abs difference of the averaged logits between the two.

    python scripts/gpu_sampler_bench.py [--scale 1.0] [--batches 20] [--host-batches 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

F_IN = 128


class _Graph:
    def __init__(self, edge_list, types, meta):
        self.edge_list, self._t, self._m = edge_list, types, meta

    def get_types(self):
        return self._t

    def get_meta_graph(self):
        return self._m


def make_graph(scale, seed=0):
    """MAG-schema graph: papers cite papers, are written by authors, have fields and a venue (years 1990-2020)."""
    rng = np.random.RandomState(seed)
    n = {"paper": int(100000 * scale), "author": int(60000 * scale), "field": int(8000 * scale), "venue": 500}
    year = rng.randint(1990, 2021, n["paper"])
    el = defaultdict(lambda: defaultdict(lambda: defaultdict(dict)))
    meta = []

    def add(tt, st, rel, tgt, src, tm):
        fwd, rev = el[tt][st][rel], el[st][tt]["rev_" + rel]
        for a, b, t in zip(tgt.tolist(), src.tolist(), tm.tolist()):
            fwd.setdefault(a, {})[b] = t
            rev.setdefault(b, {})[a] = t
        meta.extend([(tt, st, rel), (st, tt, "rev_" + rel)])

    P = n["paper"]
    # heavy-tailed citation / authorship degrees so that hubs (degree >> width) occur
    cited = (rng.pareto(1.2, 4 * P) * 50).astype(np.int64) % P
    citing = rng.randint(0, P, 4 * P)
    add("paper", "paper", "PP_cite", citing, cited, year[citing])
    pa = rng.randint(0, P, 3 * P)
    au = (rng.pareto(1.5, 3 * P) * 30).astype(np.int64) % n["author"]
    add("paper", "author", "AP_write", pa, au, year[pa])
    pf = rng.randint(0, P, 3 * P)
    fi = (rng.pareto(1.0, 3 * P) * 20).astype(np.int64) % n["field"]
    add("paper", "field", "PF_in_L2", pf, fi, year[pf])
    add("paper", "venue", "PV_Journal", np.arange(P), rng.randint(0, n["venue"], P), year)
    for t in n:                                            # 'self' relation of every type (not sampled from)
        ids = np.arange(n[t])
        rel = el[t][t]["self"]
        for i in ids.tolist():
            rel[i] = {i: None}
        meta.append((t, t, "self"))
    seen, meta_u = set(), []
    for m in meta:
        if m[2] != "self" and m not in seen:
            seen.add(m)
            meta_u.append(m)
    n_edges = sum(len(v) for a in el.values() for b in a.values() for c in b.values() for v in c.values())
    return _Graph(el, list(n), meta_u), n, year, n_edges


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:                                      # noqa: BLE001
        return [torch.cuda.get_device_name(0), "not measured"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--host-batches", type=int, default=3)
    ap.add_argument("--settings", default="6x520,3x64")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from pyhgt_b200 import data as hdata, sampler
    from pyhgt_b200.model import GNN
    import pyhgt_b200
    dev = torch.device("cuda:0")
    t0 = time.time()
    g, n, year, n_edges = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    rng = np.random.RandomState(1)
    tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_IN).astype(np.float32)) for t in n}
    dg = sampler.DeviceGraph(fg, dev, tables)
    build_s = time.time() - t0
    time_range = {y: True for y in range(1990, 2016)}
    tables_np = {t: v.numpy() for t, v in tables.items()}

    def extractor(layer_data, graph):
        feature, times, indxs = {}, {}, {}
        for t in graph.get_types():
            ids = np.fromiter(layer_data[t].keys(), dtype=np.int64) if t in layer_data else np.zeros(0, np.int64)
            feature[t] = tables_np[t][ids]
            times[t] = np.array([layer_data[t][i][1] for i in ids.tolist()], dtype=np.int64)
            indxs[t] = ids
        return feature, times, indxs, []

    def seeds(i):
        r = np.random.RandomState(100 + i)
        p = r.choice(np.nonzero(year <= 2015)[0], 128, replace=False)
        return {"paper": np.stack([p, year[p]], 1)}

    edge_dict = {e[2]: i for i, e in enumerate(g.get_meta_graph())}
    edge_dict["self"] = len(edge_dict)
    torch.manual_seed(0)
    gnn = GNN(F_IN, 512, len(n), len(edge_dict), 8, 4, 0.2, "hgt", True, False, True).to(dev).train()
    pyhgt_b200.HGTConv.keep_att = False
    name, power = card()
    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        host = []
        for i in range(args.host_batches):
            np.random.seed(i)
            torch.cuda.synchronize()
            a = time.perf_counter()
            feature, times, edge_list, _, _ = sampler.sample_subgraph(fg, time_range, depth, width, seeds(i), extractor)
            hdata.to_torch(feature, times, edge_list, g, device=dev, prebuild_plan=True)
            torch.cuda.synchronize()
            host.append((time.perf_counter() - a) * 1e3)
        gen = torch.Generator().manual_seed(0)
        for i in range(3):
            out = sampler.sample_subgraph_cuda(dg, time_range, depth, width, seeds(i), gen)
        devt = []
        for i in range(args.batches):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = sampler.sample_subgraph_cuda(dg, time_range, depth, width, seeds(i), gen)
            e1.record()
            torch.cuda.synchronize()
            devt.append(e0.elapsed_time(e1))
        per_sub = {}
        for B in (1, 8, 32):
            inps = [seeds(i) for i in range(B)]
            for _ in range(2):
                sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, gen)
            tb = []
            for i in range(max(5, args.batches // B)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, gen)
                e1.record()
                torch.cuda.synchronize()
                tb.append(e0.elapsed_time(e1) / B)
            per_sub[str(B)] = round(float(np.median(tb)), 3)
        nf, nt, etime, ei, et = out[:5]
        train = []
        for i in range(8):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = gnn(nf, nt, etime, ei, et)
            y.square().mean().backward()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                train.append(e0.elapsed_time(e1))
        print(json.dumps({"setting": {"depth": depth, "width": width, "seeds": 128},
                          "graph": {"nodes": n, "edges": n_edges, "build_s": round(build_s, 1)},
                          "batch": {"nodes": int(nt.numel()), "edges": int(ei.shape[1])},
                          "host_ms": round(float(np.median(host)), 2), "host_batches": len(host),
                          "device_ms": round(float(np.median(devt)), 3), "device_batches": len(devt),
                          "device_ms_per_subgraph": per_sub,
                          "train_fwd_bwd_ms": round(float(np.median(train)), 3),
                          "gpu": name, "power_limit": power}), flush=True)
    mask_timing(args, dg, seeds, time_range, name, power)
    vr_eval(args, dg, g, gnn, edge_dict, seeds(0), time_range, name, power)


def mask_timing(args, dg, seeds, time_range, name, power, n_seed=128):
    """The paper-field label-leak mask (OAG/train_paper_field.py:109-122) against no mask, at every setting and B = 1, 8,
    32: `edge_mask` acts inside the rebuild's count and write passes, so it should cost nothing measurable.  In this
    graph PF_in_L2 has paper as its target (OAG names the paper -> field direction rev_PF_in_L2), hence the keys.
    The two variants alternate call by call from the same generator state; CUDA events / B, median."""
    from pyhgt_b200 import sampler
    mask = {("paper", "field", "PF_in_L2"): (n_seed, 0), ("field", "paper", "rev_PF_in_L2"): (0, n_seed)}
    variants = (("none", None), ("mask", mask))
    res, edges = {}, {}
    for setting in args.settings.split(","):
        depth, width = (int(v) for v in setting.split("x"))
        per = {}
        for B in (1, 8, 32):
            inps = [seeds(i) for i in range(B)]
            tl = {label: [] for label, _ in variants}
            for i in range(2 + max(5, args.batches // B)):
                for label, m in (variants if i % 2 == 0 else variants[::-1]):
                    gen = torch.Generator().manual_seed(i)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    out = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, gen, edge_mask=m)
                    e1.record()
                    torch.cuda.synchronize()
                    if i >= 2:                                 # the first two rounds warm both variants up
                        tl[label].append(e0.elapsed_time(e1) / B)
                    if B == 1 and i == 0:
                        edges.setdefault(setting, {})[label] = int(out[0][3].shape[1])
            per[str(B)] = {label: round(float(np.median(v)), 3) for label, v in tl.items()}
        res[setting] = per
    print(json.dumps({"edge_mask": "paper-field label mask, %d paper seeds" % n_seed,
                      "device_ms_per_subgraph": res, "edges_of_one_subgraph": edges,
                      "gpu": name, "power_limit": power}), flush=True)


def vr_eval(args, dg, g, gnn, edge_dict, inp, time_range, name, power, n_vr=8, n_cls=349):
    """Variance-reduced evaluation (pyHGT ogbn-mag/eval_ogbn_mag.py:128-152): n_vr subgraphs around the same 128 seeds,
    logits of the seeds averaged.  Timed two ways from the same generator state (so the same subgraphs): n_vr single
    samples and n_vr forwards, and one batched sample + merge_batches + one forward over the union."""
    from pyhgt_b200 import sampler
    depth, width = (int(v) for v in args.settings.split(",")[0].split("x"))
    dev = dg.device
    T, R = len(dg.types), len(edge_dict)
    torch.manual_seed(1)
    head = torch.nn.Linear(512, n_cls).to(dev)
    gnn.eval()
    n_seed = inp["paper"].shape[0]

    def singles(gen):
        acc = 0
        for _ in range(n_vr):
            b = sampler.sample_subgraph_cuda(dg, time_range, depth, width, inp, gen)
            p0 = b[5]["paper"][0]
            acc = acc + head(gnn(*b[:5])[p0:p0 + n_seed])
        return acc / n_vr

    def batched(gen):
        bs = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, [inp] * n_vr, gen)
        nf, nt, etime, ei, et, rows = sampler.merge_batches(bs, T, R)
        y = gnn(nf, nt, etime, ei, et)
        sel = torch.cat([rows[v][b[5]["paper"][0]:b[5]["paper"][0] + n_seed] for v, b in enumerate(bs)])
        return head(y[sel]).view(n_vr, n_seed, n_cls).mean(0)

    times = {}
    with torch.no_grad():
        for label, fn in (("singles", singles), ("batched", batched)):
            for _ in range(2):
                fn(torch.Generator().manual_seed(0))
            tl = []
            for i in range(max(5, args.batches // 4)):
                gen = torch.Generator().manual_seed(i)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(gen)
                e1.record()
                torch.cuda.synchronize()
                tl.append(e0.elapsed_time(e1))
            times[label] = (round(float(np.median(tl)), 2), len(tl))
        diff = (singles(torch.Generator().manual_seed(7)) - batched(torch.Generator().manual_seed(7))).abs().max().item()
    gnn.train()
    print(json.dumps({"vr_eval": {"subgraphs": n_vr, "seeds": n_seed, "depth": depth, "width": width,
                                  "model": "GNN 4 layers n_hid 512 + linear head, eval, no_grad"},
                      "singles_ms": times["singles"][0], "batched_merged_ms": times["batched"][0],
                      "repeats": times["singles"][1], "max_abs_diff": diff,
                      "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
