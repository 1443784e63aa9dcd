"""24-bit against bs16 [K'|V'] / RTE gather tables, stage by stage through the C ABI, in one process.

For each benchmark graph (c2, c3, c5 of bench.py at full size) one HGTConv layer's weights are folded once; then, alternating
24-bit and bs16 tables, the script times the projection GEMM (hgt_typed_linear_t24 / hgt_typed_linear_bs16: Q as fp32
and the K'/V' blocks in the table, in one call) and the edge pass (hgt_edge_forward_t24 / _bs16, gelu(agg) as fp32) with
CUDA events, and reports the medians, the edge launch's algorithmic bytes at the table's true row size (bench.py's
roofline counts 4 bytes per table element whatever the tables hold) with the rate they imply, and the deviation of each
format's gelu(agg) from the fp32-table edge pass.  The card's name, power limit and SM clock go with each line.

    python scripts/bs16_tables_bench.py [--configs c2,c3,c5] [--reps 10]

Prints one JSON line per graph.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyhgt_b200 import HGTConv, _lib, plan as P, synth  # noqa: E402

CONFIGS = {"c2": (256, False, lambda: synth.make_mag_shaped(1.0)),
           "c3": (400, True, lambda: synth.make_oag_shaped(1.0)),
           "c5": (128, False, lambda: synth.make_powerlaw(64_000_000))}
H = 8
FORMATS = {"t24": _lib.TABLE_T24, "bs16": _lib.TABLE_BS16}


def edge_bytes(n_edges, n_dst, row, rte):
    """E * (row [K'|V'] + 4 [kv_row] (+ 4 [rte_row] + row [RTE])) + N_dst * (d*4 [Q] + d*4 [agg] + 4); row in bytes."""
    per_edge = row + 4 + ((4 + row) if rte else 0)
    return n_edges * per_edge + n_dst * 4


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


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
    ewsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(ewsb))
    ews = torch.empty(ewsb.value, dtype=torch.uint8, device=dev)
    rt = None
    if rte:
        rt = torch.empty(P.RTE_MAX_LEN, d, device=dev)
        rg = lt.rt_group
        _lib.call("hgt_typed_linear", m.emb.emb.weight.data_ptr(), d, m.emb.lin.weight.data_ptr(),
                  m.emb.lin.bias.data_ptr(), d, d, rg[0].data_ptr(), rg[1].ctypes.data, rg[2], rg[3].data_ptr(),
                  rt.data_ptr(), 1, None, 0, st)
    tr = lt.rte_groups

    def edge(sfx, q, kv, kvr, agg):
        _lib.call("hgt_edge_forward" + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr),
                  plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(), _lib.ptr(plan.rte_row) if rte else None,
                  plan.csr_eid.data_ptr(), plan.tiles.data_ptr(), plan.n_tiles, plan.n_split, plan.hubs.data_ptr(),
                  plan.n_hubs, N, E, d, H, 1, agg.data_ptr(), None, None, None, None, ews.data_ptr(), ews.numel(), 0,
                  _lib.ptr(plan.tile_counts_dev), plan.type_row0_dev.data_ptr(), T, None, st)

    # the fp32-table reference, then freed
    proj = torch.empty(lt.proj_elems, device=dev)
    proj[lt.kv_off + plan.kv_rows * 2 * d:].zero_()
    _lib.call("hgt_typed_linear", x.data_ptr(), d, w_cat.data_ptr(), b_cat.data_ptr(), d, d, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), proj.data_ptr(), 0, ws.data_ptr(), ws.numel(), st)
    kvr32 = None
    if rte:
        kvr32 = torch.zeros((npairs * P.RTE_MAX_LEN + 1) * 2 * d, device=dev)
        _lib.call("hgt_typed_linear", rt.data_ptr(), d, w_cat.data_ptr(), None, d, d, tr[0].data_ptr(),
                  tr[1].ctypes.data, tr[2], tr[3].data_ptr(), kvr32.data_ptr(), 1, None, 0, st)
    agg32 = torch.empty(N, d, device=dev)
    edge("", proj, proj[lt.kv_off:], kvr32, agg32)
    q32 = proj[:N * d].clone()
    del proj, kvr32

    tabs = {}
    for name, fmt in FORMATS.items():
        row = _lib.gather_table_row_bytes(fmt, 2 * d)
        q = torch.empty(lt.kv_off, device=dev)
        kv = torch.zeros((plan.kv_rows + 1) * row, dtype=torch.uint8, device=dev)
        kvr = None
        if rte:
            kvr = torch.zeros((npairs * P.RTE_MAX_LEN + 1) * row, dtype=torch.uint8, device=dev)
            _lib.call("hgt_typed_linear" + _lib.TABLE_SUFFIX[fmt], rt.data_ptr(), d, w_cat.data_ptr(), None, d, d,
                      tr[0].data_ptr(), tr[1].ctypes.data, tr[2], tr[3].data_ptr(), None, 0, kvr.data_ptr(), 1, None,
                      0, st)
        tabs[name] = (fmt, row, q, kv, kvr, torch.empty(N, d, device=dev))

    def project(name):
        fmt, _, q, kv, _, _ = tabs[name]
        _lib.call("hgt_typed_linear" + _lib.TABLE_SUFFIX[fmt], x.data_ptr(), d, w_cat.data_ptr(), b_cat.data_ptr(), d,
                  d, g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), q.data_ptr(), lt.kv_off,
                  kv.data_ptr(), 0, ws.data_ptr(), ws.numel(), st)

    def edge_of(name):
        fmt, _, q, kv, kvr, agg = tabs[name]
        edge(_lib.TABLE_SUFFIX[fmt], q, kv, kvr, agg)

    for name in tabs:                                          # warm-up: module loads, tensor-map templates
        project(name)
        edge_of(name)
    res = {name: {"proj": [], "edge": []} for name in tabs}
    for _ in range(reps):
        for name in tabs:
            res[name]["proj"].append(timed(lambda: project(name)))
            res[name]["edge"].append(timed(lambda: edge_of(name)))
    torch.cuda.synchronize()
    n_dst = int(((plan.row_ptr[1:] - plan.row_ptr[:-1]) > 0).sum())
    out = {"config": config, "N": N, "E": E, "d": d, "heads": H, "rte": rte, "card": card(), "reps": reps}
    for name, (fmt, row, q, kv, kvr, agg) in tabs.items():
        med = {k: sorted(v)[len(v) // 2] for k, v in res[name].items()}
        spread = {k: round((max(v) - min(v)) / med[k], 4) for k, v in res[name].items()}
        nbytes = edge_bytes(E, n_dst, row, rte) + n_dst * 2 * d * 4
        out[name] = {"row_bytes": row, "proj_ms": round(med["proj"], 3), "edge_ms": round(med["edge"], 3),
                     "spread": spread, "edge_GB": round(nbytes / 1e9, 2),
                     "edge_GBps": round(nbytes / med["edge"] / 1e6, 1),
                     "agg_max_abs": float((agg - agg32).abs().max()),
                     "agg_rel_fro": float((agg - agg32).double().norm() / agg32.double().norm()),
                     "q_equal": bool(torch.equal(q[:N * d], q32))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3,c5")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bs16_tables_bench.py needs a CUDA device")
    for c in args.configs.split(","):
        print(json.dumps(run(c, args.reps)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
