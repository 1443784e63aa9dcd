"""HGT layers and the typed GEMM under torch.set_float32_matmul_precision "highest" (split-bf16 x3) and "medium" (one
bf16 product), alternating in one process.  Prints one JSON line per round, workload and setting:
  c2 / c3 / c5 forward (one HGTConv, bench.py's graphs and widths), each with bf16 autocast off and on: median CUDA-event
      ms per forward over --steps, the `proj_linear` / `upd_linear` stage times from HGTConv.event_sink, and for "medium"
      the max-abs / relative-Frobenius deviation of the output from "highest" on the same seeded inputs;
  c4 training step (3 layers, forward + backward): median ms per step and max_memory_allocated;
  gemm: the typed GEMM alone at the C2 projection shape (K = 256; groups of 736,389 / 1,134,649 / 8,740 / 59,965 rows;
      five 256-wide column blocks), fp32 and bf16 output: P = 3 (impl 2) and P = 1 (impl 3).  The one-product kernel's
      k-block at 128 / 256 columns is 32 for fp32 A unless HGT_TC_P1_KB=64; the script measures that variant in a child
      process (--gemm-only), since the switch is read once per process.
The card name, power limit and SM clock are read in the same run.  Writes nothing.

    python scripts/matmul_precision_bench.py [--steps 10] [--warmup 3] [--rounds 2] [--scale 1.0]
"""
import argparse
import contextlib
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                # noqa: E402  (graph generator and config settings only)
from pyhgt_b200 import HGTConv, _lib        # noqa: E402
from pyhgt_b200 import plan as _plan        # noqa: E402

SETTINGS = ("highest", "medium")
C2_GROUPS = (736389, 1134649, 8740, 59965)


@contextlib.contextmanager
def _precision(p):
    old = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision(p)
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(old)


def _autocast(bf16):
    return torch.autocast("cuda", dtype=torch.bfloat16) if bf16 else contextlib.nullcontext()


def _card(dev):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader",
                            "-i", str(dev.index or 0)], capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = None
    return {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q}


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    evs[0].record()
    for i in range(steps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    ms = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(steps))
    return ms[len(ms) // 2], ms[0], ms[-1]


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
    for bf16 in (False, True):
        ref = None
        for setting in SETTINGS:
            with torch.no_grad(), _autocast(bf16), _precision(setting):
                med, lo, hi = _time(lambda: m(x, *args), steps, warmup)
                HGTConv.event_sink = []
                for _ in range(steps):
                    m(x, *args)
                torch.cuda.synchronize()
                stages = {}
                for name, a, b in HGTConv.event_sink:
                    stages.setdefault(name, []).append(a.elapsed_time(b))
                HGTConv.event_sink = None
                out = m(x, *args)
            st = {k: sorted(v)[len(v) // 2] for k, v in stages.items()}
            line = dict(card, round=rnd, config=config, bf16_autocast=bf16, precision=setting,
                        workload="%s: N=%d, E=%d, d=%d, H=%d, rte=%s" % (cfg["label"], N, E, d, H, rte),
                        ms_per_forward=med, min_ms=lo, max_ms=hi, proj_linear_ms=st.get("proj_linear"),
                        upd_linear_ms=st.get("upd_linear"), edge_ms=st.get("edge"))
            if ref is None:
                ref = out
            else:
                diff = (out - ref).double()
                line["max_abs_vs_highest"] = float(diff.abs().max())
                line["rel_fro_vs_highest"] = float(diff.norm() / ref.double().norm())
            print(json.dumps(line), flush=True)
            del out
        del ref
    del m, x


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

    def step():
        layers.zero_grad(set_to_none=True)
        h = x
        for m in layers:
            h = m(h, nt, ei, et)
        (h * w).sum().backward()

    for setting in SETTINGS:
        with _precision(setting):
            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            med, lo, hi = _time(step, steps, 0)
        print(json.dumps(dict(card, round=rnd, config="c4", precision=setting,
                              workload="%s: N=%d, E=%d, d=%d, H=%d, %d layers" % (cfg["label"], N, E, D, H, L),
                              ms_per_step=med, min_ms=lo, max_ms=hi,
                              max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))), flush=True)
    del layers


def gemm_lines(steps, warmup, rnd, dev, card, variant):
    """The C2 projection GEMM alone: impl 2 (P = 3) and impl 3 (P = 1), fp32 and bf16 output."""
    K = width = 256
    ncb = 5
    groups, cblocks, a0, out0 = [], [], 0, 0
    for g, m in enumerate(C2_GROUPS):
        groups.append((a0, m, g * ncb * width, ncb, len(cblocks), 1))
        cblocks += [(out0 + cb * width, ncb * width) for cb in range(ncb)]
        a0 += m
        out0 += m * ncb * width
    tab = _plan._pack_groups(groups, cblocks, dev)
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator(device=dev).manual_seed(0)
    a = torch.randn(a0, K, device=dev, generator=gen)
    w = torch.randn(len(C2_GROUPS) * ncb * width, K, device=dev, generator=gen)
    b = torch.randn(w.shape[0], device=dev, generator=gen)
    st = torch.cuda.current_stream().cuda_stream
    flops = 2.0 * a0 * ncb * width * K
    for dtype in (torch.float32, torch.bfloat16):
        out = torch.empty(out0, dtype=dtype, device=dev)
        for impl in ((3,) if variant == "kb64" else (2, 3)):
            wsb = ctypes.c_size_t()
            _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
            ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
            fn = "hgt_typed_linear_bf16" if dtype == torch.bfloat16 else "hgt_typed_linear"
            med, lo, hi = _time(lambda: _lib.call(fn, a.data_ptr(), K, w.data_ptr(), b.data_ptr(), K, width,
                                                  g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(),
                                                  out.data_ptr(), impl, ws.data_ptr(), ws.numel(), st), steps, warmup)
            print(json.dumps(dict(card, round=rnd, config="gemm_c2_projection", out_dtype=str(dtype).split(".")[1],
                                  products=1 if impl == 3 else 3,
                                  p1_kblock=(64 if variant == "kb64" else 32) if impl == 3 else None,
                                  workspace_gb=round(wsb.value / 1e9, 2), ms=med, min_ms=lo, max_ms=hi,
                                  tflops_per_product=round(flops / (med / 1e3) / 1e12, 1),
                                  out_gb=round(out.numel() * out.element_size() / 1e9, 2))), flush=True)
            del ws
        del out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--configs", default="gemm,c2,c3,c5,c4")
    ap.add_argument("--gemm-only", action="store_true", help="only the GEMM lines (used for the HGT_TC_P1_KB=64 child)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("matmul_precision_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = _card(dev)
    variant = "kb64" if os.environ.get("HGT_TC_P1_KB") == "64" else "kb32"
    for rnd in range(args.rounds):
        for config in (["gemm"] if args.gemm_only else args.configs.split(",")):
            if config == "gemm":
                gemm_lines(args.steps, args.warmup, rnd, dev, card, variant)
                if not args.gemm_only:
                    env = dict(os.environ, HGT_TC_P1_KB="64")
                    subprocess.run([sys.executable, os.path.abspath(__file__), "--gemm-only", "--rounds", "1",
                                    "--steps", str(args.steps), "--warmup", str(args.warmup)], env=env, check=True)
            elif config == "c4":
                train_lines(args.scale, args.steps, args.warmup, rnd, dev, card)
            else:
                forward_lines(config, args.scale, args.steps, args.warmup, rnd, dev, card)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
