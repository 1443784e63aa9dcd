"""float32 vs bf16 node features on device-sampled subgraphs: sampler, input adapter, eager and graphed training step.

Workload: the MAG-schema graph of gpu_sampler_bench.make_graph with feature tables of width F (128: ogbn-mag's input
width; 1169: OAG's), stored in bf16 (DeviceGraph(..., feature_dtype=torch.bfloat16)), 128 paper seeds per subgraph at
the ogbn-mag recipe setting (depth 6, width 520).  An epoch is the 32 subgraphs of ONE sample_subgraphs_cuda call.  The
float32 variant widens the stored rows into float32 batches (the default); the bf16 variant keeps them
(feature_dtype=torch.bfloat16) and the adapter GEMM reads them as its bf16 operand.  Model and recipe as in
graphed_train_bench.py (GNN(F -> 512, 4 HGT layers, 8 heads, RTE, dropout 0.2), AdamW + OneCycleLR + clip 1.0); both
variants start from the same weights.

The variants alternate (--epochs of each, each epoch sampled afresh from the same seeds).  Per variant, medians with
min-max over its epochs of:
  sampler_ms_per_subgraph   one sample_subgraphs_cuda call / 32 (host clock ending in a device synchronise)
  adapter_fwd_ms, adapter_bwd_ms   the input adapter alone (GNN._adapter_autograd and the backward of its output),
                            CUDA events, per subgraph
  eager_step_ms, graphed_step_ms   one training step per subgraph, eager and replayed by GraphedTrainStep (per-variant
                            signature: the epoch's per-type maximum), host clock ending in a device synchronise
  max_memory_allocated_mb   torch.cuda.max_memory_allocated over the variant's eager epoch
  batch_feature_mb          the node_feature bytes of the epoch's 32 subgraphs
One JSON line per (F, variant), with the card's name and power limit.

    python scripts/bf16_features_bench.py [--scale 1.0] [--epochs 3] [--widths 128,1169] [--setting 6x520]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_sampler_bench import card, make_graph  # noqa: E402
from graphed_train_bench import BATCHES, N_CLS, recipe  # noqa: E402

BF16 = torch.bfloat16


class Model(torch.nn.Module):
    def __init__(self, F_in, T, R, dropout):
        super().__init__()
        from pyhgt_b200.model import GNN
        self.gnn = GNN(F_in, 512, T, R, 8, 4, dropout, "hgt", True, True, True)
        self.head = torch.nn.Linear(512, N_CLS)

    def loss(self, x, nt, tm, ei, et, y, r0):
        h = self.gnn(x, nt, tm, ei, et)[r0:r0 + y.shape[0]]
        return torch.nn.functional.nll_loss(torch.nn.functional.log_softmax(self.head(h), -1), y, ignore_index=-100)


def sample(dg, time_range, depth, width, year, paper_label, dtype):
    from pyhgt_b200 import plan as P, sampler
    rng = np.random.RandomState(0)
    pool = np.nonzero(year <= 2015)[0]
    inps = []
    for _ in range(BATCHES):
        p = rng.choice(pool, 128, replace=False)
        inps.append({"paper": np.stack([p, year[p]], 1)})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    members = sampler.sample_subgraphs_cuda(dg, time_range, depth, width, inps, torch.Generator().manual_seed(0),
                                            feature_dtype=dtype)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / BATCHES
    out = []
    for m, inp in zip(members, inps):
        y = torch.from_numpy(paper_label[inp["paper"][:, 0]]).to(dg.device)
        p0 = P.get_plan(m[1], m[3], m[4], m[2], len(dg.types), len(dg.edge_dict)).type_row0[dg.slot["paper"]]
        out.append((m[:5], y, p0))
    return out, ms


def adapter_ms(model, batches):
    """Forward and backward of the input adapter alone, per subgraph (CUDA events)."""
    from pyhgt_b200 import plan as P
    gnn = model.gnn
    T, R = gnn.num_types, gnn.gcs[0].base_conv.num_relations
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    fwd = bwd = 0.0
    for (nf, nt, tm, ei, et), _, _ in batches:
        plan = P.get_plan(nt, ei, et, tm, T, R)
        ev[0].record()
        res = gnn._adapter_autograd(nf, plan)
        ev[1].record()
        res.backward(torch.ones_like(res))
        ev[2].record()
        torch.cuda.synchronize()
        fwd += ev[0].elapsed_time(ev[1])
        bwd += ev[1].elapsed_time(ev[2])
    model.zero_grad(set_to_none=True)
    return fwd / len(batches), bwd / len(batches)


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / BATCHES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--widths", default="128,1169")
    ap.add_argument("--setting", default="6x520")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import copy

    import pyhgt_b200
    from pyhgt_b200 import graphed, plan as P, sampler
    dev = torch.device("cuda:0")
    P._CACHE_SIZE = 2 * BATCHES + 8
    pyhgt_b200.HGTConv.keep_att = False
    depth, width = (int(v) for v in args.setting.split("x"))
    g, n, year, _ = make_graph(args.scale)
    fg = sampler.FrozenGraph(g)
    name, power = card()
    for F_in in (int(v) for v in args.widths.split(",")):
        rng = np.random.RandomState(1)
        tables = {t: torch.from_numpy(rng.randn(max(fg.n_ids.get(t, 1), 1), F_in).astype(np.float32)) for t in n}
        dg = sampler.DeviceGraph(fg, dev, tables, feature_dtype=BF16)
        del tables
        paper_label = rng.randint(0, N_CLS, n["paper"]).astype(np.int64)
        time_range = {y: True for y in range(1990, 2016)}
        T, R = len(dg.types), len(dg.edge_dict)
        paper = dg.slot["paper"]
        torch.manual_seed(0)
        base = Model(F_in, T, R, 0.2).to(dev).train()
        variants = {}
        for key, dtype in (("float32", torch.float32), ("bf16", BF16)):
            model = copy.deepcopy(base)
            opt, sched = recipe(model, 10 ** 6)
            batches, _ = sample(dg, time_range, depth, width, year, paper_label, dtype)
            plans = [P.get_plan(b[1], b[3], b[4], b[2], T, R) for b, _, _ in batches]
            sig = graphed.GraphSignature([max(p.type_count[t] for p in plans) for t in range(T)],
                                         max(p.n_edges for p in plans), {pr for p in plans for pr in p.pairs}, R, F_in,
                                         feat_dtype=dtype)
            r0 = int(sig.row0[paper])
            m_g = copy.deepcopy(base)
            opt_g, sched_g = recipe(m_g, 10 ** 6)
            step = graphed.GraphedTrainStep(lambda x, nt, tm, ei, et, tg, m=m_g: m.loss(x, nt, tm, ei, et, tg[paper], r0),
                                            sig, dev, optimizer=opt_g, clip_norm=1.0,
                                            targets={paper: ((), torch.int64, -100)})
            variants[key] = dict(dtype=dtype, model=model, opt=opt, sched=sched, step=step, sched_g=sched_g,
                                 rows={k: [] for k in ("sampler_ms_per_subgraph", "adapter_fwd_ms", "adapter_bwd_ms",
                                                       "eager_step_ms", "graphed_step_ms", "max_memory_allocated_mb",
                                                       "batch_feature_mb")})
            (nf, nt, tm, ei, et), y, _ = batches[0]
            step(nf, nt, tm, ei, et, targets={paper: y})                # capture outside the timed epochs
        for ep in range(args.epochs + 1):                               # epoch 0 warms up every shape
            for key, v in variants.items():
                batches, s_ms = sample(dg, time_range, depth, width, year, paper_label, v["dtype"])
                model, opt, sched = v["model"], v["opt"], v["sched"]
                a_f, a_b = adapter_ms(model, batches)

                def eager():
                    for (nf, nt, tm, ei, et), y, p0 in batches:
                        loss = model.loss(nf, nt, tm, ei, et, y, p0)
                        opt.zero_grad()
                        loss.backward()
                        torch.nn.utils.clip_grad_norm_([p for g_ in opt.param_groups for p in g_["params"]], 1.0,
                                                       foreach=True)
                        opt.step()
                        sched.step()

                def replay():
                    for (nf, nt, tm, ei, et), y, _ in batches:
                        v["step"](nf, nt, tm, ei, et, targets={paper: y})
                        v["sched_g"].step()

                torch.cuda.reset_peak_memory_stats()
                e_ms = host_ms(eager)
                peak = torch.cuda.max_memory_allocated() / 2 ** 20
                g_ms = host_ms(replay)
                fbytes = sum(b[0][0].numel() * b[0][0].element_size() for b in batches) / 2 ** 20
                if ep == 0:
                    continue
                for k, val in (("sampler_ms_per_subgraph", s_ms), ("adapter_fwd_ms", a_f), ("adapter_bwd_ms", a_b),
                               ("eager_step_ms", e_ms), ("graphed_step_ms", g_ms), ("max_memory_allocated_mb", peak),
                               ("batch_feature_mb", fbytes)):
                    v["rows"][k].append(val)
                del batches
        for key, v in variants.items():
            stats = {k: {"median": round(float(np.median(x)), 4), "min": round(float(np.min(x)), 4),
                         "max": round(float(np.max(x)), 4)} for k, x in v["rows"].items()}
            print(json.dumps({"in_dim": F_in, "variant": key, "setting": {"depth": depth, "width": width, "seeds": 128,
                                                                          "batches_per_epoch": BATCHES},
                              "epochs": args.epochs, **stats, "gpu": name, "power_limit": power}), flush=True)
        del variants, dg, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
