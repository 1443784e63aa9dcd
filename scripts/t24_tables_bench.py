"""fp32 against 24-bit [K'|V'] / RTE gather tables, stage by stage through the C ABI, in one process.

For each benchmark graph (c2, c3, c5 of bench.py at full size) one HGTConv layer's weights are folded once; then, alternating
fp32 and 24-bit tables, the script times the projection GEMM (hgt_typed_linear into the fp32 [Q | K'|V'] buffer, or
hgt_typed_linear_t24: Q as fp32 and the K'/V' blocks as 24-bit, in one call) and the edge pass (hgt_edge_forward /
hgt_edge_forward_t24, gelu(agg) as fp32) with CUDA events, and reports the medians, the edge launch's algorithmic bytes
at the table's true element size (bench.py's roofline counts 4 bytes per table element whatever the tables hold) with the
rate they imply, and the deviation of the edge output.

    python scripts/t24_tables_bench.py [--configs c2,c3,c5] [--reps 10]

Prints one JSON line per graph.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyhgt_b200 import HGTConv, _lib, plan as P, synth  # noqa: E402

CONFIGS = {"c2": (256, False, lambda: synth.make_mag_shaped(1.0)),
           "c3": (400, True, lambda: synth.make_oag_shaped(1.0)),
           "c5": (128, False, lambda: synth.make_powerlaw(64_000_000))}
H = 8


def edge_bytes(n_edges, n_dst, d, s_kv, rte):
    """E * (2 d s_kv [K'|V' row] + 4 [kv_row] (+ 4 [rte_row] + 2 d s_kv [RTE row])) + N_dst * (d*4 [Q] + d*4 [agg] + 4)."""
    per_edge = 2 * d * s_kv + 4 + ((4 + 2 * d * s_kv) if rte else 0)
    return n_edges * per_edge + n_dst * (2 * d * 4 + 4)


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2]


def run(config, reps):
    dev = torch.device("cuda:0")
    d, rte, make = CONFIGS[config]
    g = make()
    torch.manual_seed(0)
    m = HGTConv(d, d, g.num_types, g.num_relations, H, 0.0, True, rte).to(dev).eval()
    T, R = g.num_types, g.num_relations
    plan = P.build_plan(g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev),
                        g.edge_time.to(dev) if rte else None, T, R)
    lt = P.layer_tables(plan, d, d)
    N, E, npairs = plan.n_nodes, plan.n_edges, plan.n_pairs
    x = torch.randn(N, d, generator=torch.Generator().manual_seed(1)).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    w_cat = torch.empty(lt.cat_rows, d, device=dev)
    b_cat = torch.empty(lt.cat_rows, device=dev)
    ptr = [m._ptrs(n, [getattr(l, a) for l in ls], dev).data_ptr() for n, ls, a in (
        ("wq", m.q_linears, "weight"), ("bq", m.q_linears, "bias"), ("wk", m.k_linears, "weight"),
        ("bk", m.k_linears, "bias"), ("wv", m.v_linears, "weight"), ("bv", m.v_linears, "bias"))]
    _lib.call("hgt_fold_weights", *ptr, m.relation_att.data_ptr(), m.relation_msg.data_ptr(),
              m.relation_pri.data_ptr(), T, R, H, d, d, npairs, plan.pair_type_dev.data_ptr(),
              plan.pair_rel_dev.data_ptr(), lt.cat_row0_dev.data_ptr(), lt.q_row0_dev.data_ptr(), w_cat.data_ptr(),
              b_cat.data_ptr(), st)
    g_dev, g_host, n_g, c_dev = lt.proj_groups
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, d, d, 0, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    proj = torch.empty(lt.proj_elems, device=dev)
    q24 = torch.empty(lt.kv_off, device=dev)
    kv24 = torch.empty((plan.kv_rows + 1) * 6 * d, dtype=torch.uint8, device=dev)
    proj[lt.kv_off + plan.kv_rows * 2 * d:].zero_()
    kv24[plan.kv_rows * 6 * d:].zero_()
    kvr32 = kvr24 = None
    if rte:
        rt = torch.empty(P.RTE_MAX_LEN, d, device=dev)
        rg = lt.rt_group
        _lib.call("hgt_typed_linear", m.emb.emb.weight.data_ptr(), d, m.emb.lin.weight.data_ptr(),
                  m.emb.lin.bias.data_ptr(), d, d, rg[0].data_ptr(), rg[1].ctypes.data, rg[2], rg[3].data_ptr(),
                  rt.data_ptr(), 1, None, 0, st)
        kvr32 = torch.zeros((npairs * P.RTE_MAX_LEN + 1) * 2 * d, device=dev)
        kvr24 = torch.zeros((npairs * P.RTE_MAX_LEN + 1) * 6 * d, dtype=torch.uint8, device=dev)
        t = lt.rte_groups
        _lib.call("hgt_typed_linear", rt.data_ptr(), d, w_cat.data_ptr(), None, d, d, t[0].data_ptr(), t[1].ctypes.data,
                  t[2], t[3].data_ptr(), kvr32.data_ptr(), 1, None, 0, st)
        _lib.call("hgt_typed_linear_t24", rt.data_ptr(), d, w_cat.data_ptr(), None, d, d, t[0].data_ptr(),
                  t[1].ctypes.data, t[2], t[3].data_ptr(), None, 0, kvr24.data_ptr(), 1, None, 0, st)
    ewsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(ewsb))
    ews = torch.empty(ewsb.value, dtype=torch.uint8, device=dev)
    agg32 = torch.empty(N, d, device=dev)
    agg24 = torch.empty(N, d, device=dev)

    def project(t24):
        if t24:
            _lib.call("hgt_typed_linear_t24", x.data_ptr(), d, w_cat.data_ptr(), b_cat.data_ptr(), d, d,
                      g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), q24.data_ptr(), lt.kv_off,
                      kv24.data_ptr(), 0, ws.data_ptr(), ws.numel(), st)
        else:
            _lib.call("hgt_typed_linear", x.data_ptr(), d, w_cat.data_ptr(), b_cat.data_ptr(), d, d, g_dev.data_ptr(),
                      g_host.ctypes.data, n_g, c_dev.data_ptr(), proj.data_ptr(), 0, ws.data_ptr(), ws.numel(), st)

    def edge(t24):
        q, kv, kvr, agg = ((q24, kv24, kvr24, agg24) if t24 else (proj, proj[lt.kv_off:], kvr32, agg32))
        _lib.call("hgt_edge_forward_t24" if t24 else "hgt_edge_forward", q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr),
                  plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(), _lib.ptr(plan.rte_row) if rte else None,
                  plan.csr_eid.data_ptr(), plan.tiles.data_ptr(), plan.n_tiles, plan.n_split, plan.hubs.data_ptr(),
                  plan.n_hubs, N, E, d, H, 1, agg.data_ptr(), None, None, None, None, ews.data_ptr(), ews.numel(), 0,
                  _lib.ptr(plan.tile_counts_dev), plan.type_row0_dev.data_ptr(), T, None, st)

    for t24 in (False, True):                                  # warm-up: module loads, tensor-map templates
        project(t24)
        edge(t24)
    res = {False: {"proj": [], "edge": []}, True: {"proj": [], "edge": []}}
    for _ in range(reps):
        for t24 in (False, True):
            res[t24]["proj"].append(timed(lambda: project(t24), 1))
            res[t24]["edge"].append(timed(lambda: edge(t24), 1))
    torch.cuda.synchronize()
    n_dst = int(((plan.row_ptr[1:] - plan.row_ptr[:-1]) > 0).sum())
    out = {"config": config, "N": N, "E": E, "d": d, "heads": H, "rte": rte,
           "gpu": torch.cuda.get_device_name(0), "reps": reps}
    for t24, name, s_kv in ((False, "fp32", 4), (True, "t24", 3)):
        med = {k: sorted(v)[len(v) // 2] for k, v in res[t24].items()}
        nbytes = edge_bytes(E, n_dst, d, s_kv, rte)
        out[name] = {"proj_ms": round(med["proj"], 3), "edge_ms": round(med["edge"], 3), "edge_bytes": nbytes,
                     "edge_GBps": round(nbytes / med["edge"] / 1e6, 1)}
    diff = (agg24 - agg32).abs()
    out["agg_max_abs"] = float(diff.max())
    out["agg_rel_fro"] = float((agg24 - agg32).double().norm() / agg32.double().norm())
    out["q_equal"] = bool(torch.equal(q24[:N * d], proj[:N * d]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3,c5")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("t24_tables_bench.py needs a CUDA device")
    for c in args.configs.split(","):
        print(json.dumps(run(c, args.reps)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
