"""bf16 gather tables under torch.autocast(dtype=torch.bfloat16): the bf16-output typed GEMM, the edge forward / backward on
bf16 [K'|V'] and RTE tables, the layers that use them, and the switch that selects them.

What each deliberate fault is caught by (the edge tests are in tests/test_gpu_edge_instances.py):
  truncation instead of round-to-nearest-even in the GEMM epilogue   test_gemm_bf16_output_equals_rounded_fp32
  fp32 row stride in the bf16 gather                                 test_edge_forward_matches_fp64 (dtype bf16)
  the RTE table read as fp32 in the backward                         test_edge_backward_matches_fp64 (bf16, rte=True)
"""
import ctypes
import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, plan as P, synth          # noqa: E402
from tests.test_gpu_edge_instances import _edge_ref    # noqa: E402

BF16 = torch.bfloat16
# Deviation of a layer's output from the fp32 path with bf16 tables (8-bit mantissa of K' / V'): max-abs over LayerNorm'd
# outputs and relative Frobenius.  DESIGN.md §5.1 records the measured values these bounds come from.
OUT_MAX_ABS, OUT_REL_FRO = 5e-2, 1e-2


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(got, ref):
    return float((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-30))


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


# ---------------------------------------------------------------------------------------------------------------------
# 1. typed GEMM with a bf16 output

def _gemm_table(K, width, ms, shared_rows):
    """Groups of m rows with two column blocks each, laid out like the [K'|V'] table (ld = 2 * width).  shared_rows: every
    group reads rows [0, m) of A (the RTE tables' overlapping groups)."""
    groups, cblocks, a0, out0 = [], [], 0, 0
    for g, m in enumerate(ms):
        groups.append((0 if shared_rows else a0, m, 2 * g * width, 2, len(cblocks), g % 3 != 2))
        cblocks += [(out0, 2 * width), (out0 + width, 2 * width)]
        a0 += m
        out0 += m * 2 * width
    rows = max(ms) if shared_rows else a0
    return P._pack_groups(groups, cblocks, _dev()), rows, out0, 2 * len(ms) * width


@pytest.mark.parametrize("path,K,width,ms,shared", [
    ("tc", 64, 64, [200, 37, 128], False),           # BN = 64
    ("tc", 96, 128, [300, 129], False),              # BN = 128
    ("tc", 128, 256, [150, 257], False),             # BN = 256
    ("tc", 64, 400, [333, 64], False),               # d = 400: two 256-wide tiles, the second masked
    ("tc", 64, 64, [17 + 5 * i for i in range(70)], False),   # more than 64 groups: chunked launches
    ("presplit", 64, 64, [200, 37, 128], False),
    ("presplit", 128, 256, [150, 257], False),
    ("presplit", 64, 400, [333, 64], False),
    ("presplit", 64, 64, [17 + 5 * i for i in range(70)], False),
    ("simt", 64, 64, [240, 240, 240], True),         # RTE tables: overlapping groups on the SIMT kernel
    ("simt", 50, 100, [240, 240], True),
])
def test_gemm_bf16_output_equals_rounded_fp32(path, K, width, ms, shared):
    dev = _dev()
    tab, rows, out_elems, w_rows = _gemm_table(K, width, ms, shared)
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator().manual_seed(K + width + len(ms))
    a = (torch.randn(rows, K, generator=gen) * 3).to(dev)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    out32 = torch.zeros(out_elems, device=dev)
    out16 = torch.zeros(out_elems, dtype=BF16, device=dev)
    wsb = ctypes.c_size_t()
    if path == "presplit":
        hi = torch.empty(rows, K, dtype=BF16, device=dev)
        lo = torch.empty(rows, K, dtype=BF16, device=dev)
        _lib.call("hgt_act_split", a.data_ptr(), K, rows, K, 0, None, hi.data_ptr(), lo.data_ptr(), _st())
        _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, out in (("hgt_typed_linear_presplit", out32), ("hgt_typed_linear_presplit_bf16", out16)):
            _lib.call(fn, hi.data_ptr(), lo.data_ptr(), w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(),
                      g_host.ctypes.data, n_g, c_dev.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), _st())
    else:
        impl = 2 if path == "tc" else 1
        _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, out in (("hgt_typed_linear", out32), ("hgt_typed_linear_bf16", out16)):
            _lib.call(fn, a.data_ptr(), K, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data,
                      n_g, c_dev.data_ptr(), out.data_ptr(), impl, ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    assert out32.abs().max() > 0
    assert torch.equal(out16.view(torch.int16), out32.to(BF16).view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# 2. / 3. the edge forward and backward on bf16 tables against float64: tests/test_gpu_edge_instances.py, with the fp32
# tables, at every <VEC, NCH> instance

# ---------------------------------------------------------------------------------------------------------------------
# 4. layers under bf16 autocast

def _conv(fx, dev):
    import pyhgt_b200
    c = fx["cfg"]
    m = pyhgt_b200.HGTConv(c["in_dim"], c["out_dim"], c["num_types"], c["num_relations"], c["n_heads"], 0.0,
                           c["use_norm"], c["use_RTE"]).to(dev).eval()
    m.load_state_dict(fx["state_dict"])
    return m


def _inputs(fx, dev):
    return (fx["node_inp"].to(dev), fx["node_type"].to(dev), fx["edge_index"].to(dev), fx["edge_type"].to(dev),
            fx["edge_time"].to(dev))


def _close_to_fp32(got, ref, what):
    assert got.dtype == torch.float32 and torch.isfinite(got).all(), what
    err, fro = float((got - ref).abs().max()), _rel(got, ref)
    assert err <= OUT_MAX_ABS and fro <= OUT_REL_FRO, "%s: max-abs %.3g, rel-Frobenius %.3g vs fp32" % (what, err, fro)


def test_conv_fixture_under_bf16_autocast(conv_fixture):
    """The layer's edge stage equals float64 on its own bf16 tables, widened; its output stays close to the fp32 path."""
    fx, dev = conv_fixture, _dev()
    m = _conv(fx, dev)
    args = _inputs(fx, dev)
    with torch.no_grad():
        ref = m(*args)
        with torch.autocast("cuda", dtype=BF16):
            out = m(*args)
            _, _, c = m._forward_impl(*args, want_att=False, save=True)
    _close_to_fp32(out, ref, fx["name"])
    assert c["kv"].dtype == BF16 and (c["kvr"] is None or c["kvr"].dtype == BF16) and c["q"].dtype == torch.float32
    plan, d = c["plan"], m.out_dim
    kvr = None if c["kvr"] is None else c["kvr"].view(-1, 2 * d).cpu().double()
    agg_ref, _, _, _ = _edge_ref(plan, c["q"].view(-1, d).cpu().double(), c["kv"].view(-1, 2 * d).cpu().double(), kvr,
                                 m.n_heads)
    torch.testing.assert_close(c["agg"].cpu().double(), agg_ref, rtol=1e-4, atol=1e-5)


def test_conv_training_step_under_bf16_autocast(conv_fixture):
    fx, dev = conv_fixture, _dev()
    m = _conv(fx, dev).train()
    args = _inputs(fx, dev)
    w = torch.randn(fx["node_inp"].shape[0], m.out_dim, generator=torch.Generator().manual_seed(3)).to(dev)
    grads = []
    for bf16 in (False, True):
        m.zero_grad(set_to_none=True)
        x = args[0].clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=BF16, enabled=bf16):
            out = m(x, *args[1:])
        (out * w).sum().backward()
        grads.append([x.grad] + [p.grad for p in m.parameters()])
        if bf16:
            _close_to_fp32(out.detach(), ref_out, fx["name"] + " training forward")
        ref_out = out.detach()
    for g32, g16 in zip(*grads):
        if g32 is None:
            continue
        assert g16.dtype == torch.float32 and torch.isfinite(g16).all()
        assert _rel(g16, g32) <= 5e-2, "gradient rel-Frobenius %.3g vs fp32" % _rel(g16, g32)


@pytest.mark.parametrize("kind", ["hgt", "dense_hgt"])
def test_gnn_stack_under_bf16_autocast(kind):
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R = 3, 4
    g = synth.make_random(700, 5000, T, R, seed=4, self_loops=20)
    x = torch.randn(700, 48, generator=torch.Generator().manual_seed(1)).to(dev)
    args = (g.node_type.to(dev), g.edge_time.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
    torch.manual_seed(0)
    gnn = GNN(48, 64, T, R, 4, 3, 0.0, kind, True, True, True).to(dev)
    with torch.no_grad():
        ref = gnn(x, *args)
        with torch.autocast("cuda", dtype=BF16):
            out = gnn(x, *args)
    _close_to_fp32(out, ref, kind + " inference")
    grads = []
    for bf16 in (False, True):
        gnn.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=BF16, enabled=bf16):
            y = gnn(x, *args)
        y.square().mean().backward()
        grads.append([p.grad for p in gnn.parameters()])
        if bf16:
            _close_to_fp32(y.detach(), ref, kind + " training forward")
    for g32, g16 in zip(*grads):
        if g32 is not None:
            assert g16.dtype == torch.float32 and _rel(g16, g32) <= 5e-2


def test_sharded_local_forward_under_bf16_autocast():
    """test_sharded_local_forward_matches_full_graph's setting under autocast: one rank's shard (active prefix, owned-order
    output, compacted K'/V' runs) reproduces the full-graph bf16 result on the owned rows."""
    import pyhgt_b200
    from pyhgt_b200 import sharded
    dev = _dev()
    g = synth.make_random(900, 9000, 3, 4, seed=11, isolated_frac=0.2, self_loops=60, duplicate_edges=90)
    torch.manual_seed(5)
    m = pyhgt_b200.HGTConv(64, 64, 3, 4, 4, 0.2, True, True).to(dev).eval()
    x = torch.randn(g.num_nodes, 64)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    with torch.no_grad():
        ref = m(x.to(dev), *args).cpu()
        with torch.autocast("cuda", dtype=BF16):
            full = m(x.to(dev), *args).cpu()
    _close_to_fp32(full, ref, "full graph")
    for rank in range(2):
        sh = sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, 3, 4, rank, 2, dev)
        x_local = x[sh.local_global].to(dev)
        om = torch.full((sh.n_owned + sh.n_halo,), -1, dtype=torch.int32, device=dev)
        om[sh.own_rows] = torch.arange(sh.n_owned, dtype=torch.int32, device=dev)
        for kv_runs in (None, sh.kv_runs):
            with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
                out, _, _ = m._forward_impl(x_local, sh.node_type, sh.edge_index, sh.edge_type, sh.edge_time,
                                            want_att=False, save=False, active_per_type=sh.active_per_type,
                                            out_map=om, out_rows=sh.n_owned, kv_runs=kv_runs)
            torch.testing.assert_close(out.cpu(), full[sh.owned_global], rtol=1e-3, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# 5. the switch

@pytest.mark.parametrize("mode", ["off", "fp16", "bf16"])
def test_autocast_selects_the_entry_points(mode, monkeypatch):
    from tests.conftest import load_golden
    fx, dev = load_golden("c1_rte"), _dev()
    m = _conv(fx, dev)
    args = _inputs(fx, dev)
    w = torch.randn(fx["node_inp"].shape[0], m.out_dim, generator=torch.Generator().manual_seed(3)).to(dev)

    def run():
        with torch.no_grad():
            out = m(*args)
        m.train()
        m.zero_grad(set_to_none=True)
        x = args[0].clone().requires_grad_(True)
        y = m(x, *args[1:])
        (y * w).sum().backward()
        m.eval()
        return out, y.detach(), x.grad

    plain = run()
    names = []
    real = _lib.call

    def spy(name, *a):
        names.append(name)
        return real(name, *a)

    monkeypatch.setattr(_lib, "call", spy)
    ctx = contextlib.nullcontext() if mode == "off" else torch.autocast(
        "cuda", dtype=torch.float16 if mode == "fp16" else BF16)
    with _deterministic(True):
        with ctx:
            got = run()
    used = set(names)
    if mode == "bf16":
        assert {"hgt_edge_forward_bf16", "hgt_typed_linear_presplit_bf16", "hgt_edge_backward_dst_bf16"} <= used
        assert not used & {"hgt_edge_forward", "hgt_edge_backward", "hgt_edge_backward_dst", "hgt_edge_backward_rows",
                           "hgt_conv_forward"}
    else:
        assert not any(n.endswith("_bf16") for n in used)
        with _deterministic(True):
            again = run()
        for a, b in zip(got, again):
            assert torch.equal(a, b)
        assert torch.equal(got[0], plain[0]) and torch.equal(got[1], plain[1])


# ---------------------------------------------------------------------------------------------------------------------
# 6. sync-free batches and CUDA graphs

def test_sync_free_batch_under_bf16_autocast():
    import pyhgt_b200
    from pyhgt_b200 import data as hdata
    from tests.conftest import load_golden
    from tests.test_data_ingest import _GraphStub
    dev = _dev()
    fx = load_golden("to_torch")
    g = _GraphStub(fx["types"], fx["meta_graph"])
    T = len(fx["types"])
    d = fx["node_feature"].shape[1]

    def batch():
        nf, nt, etime, ei, et, node_dict, edge_dict = hdata.to_torch(fx["feature"], fx["time"], fx["edge_list"], g,
                                                                    device=dev, prebuild_plan=True)
        return nf, nt, etime, ei, et, len(edge_dict)

    nf, nt, etime, ei, et, R = batch()
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, T, R, 1, 0.0, True, False).to(dev).train()
    m.keep_att = False

    def step(nf, nt, ei, et):
        m.zero_grad(set_to_none=True)
        xg = nf.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=BF16):
            y = m(xg, nt, ei, et)
        y.square().sum().backward()
        with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
            z = m(nf, nt, ei, et)
        return xg.grad, z

    with _deterministic(True):
        ref = step(nf, nt, ei, et)
        torch.cuda.synchronize()
        P.clear_plan_cache()
        nf2, nt2, etime2, ei2, et2, _ = batch()
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = step(nf2, nt2, ei2, et2)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1])


def test_graphed_forward_and_train_step_under_bf16_autocast():
    from pyhgt_b200 import graphed
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R, F_IN = 3, 4, 48
    batches = [synth.make_random(n, e, T, R, seed=s, sorted_types=True, self_loops=20)
               for n, e, s in ((400, 3000, 1), (310, 2200, 2))]
    counts = [max(int((b.node_type == t).sum()) for b in batches) + 5 for t in range(T)]
    pairs = {(int(b.node_type[s_]), int(r_)) for b in batches
             for s_, r_ in zip(b.edge_index[0].tolist(), b.edge_type.tolist())}
    sig = graphed.GraphSignature(counts, max(b.edge_type.numel() for b in batches) + 100, pairs, R, F_IN)
    torch.manual_seed(11)
    gnn = GNN(F_IN, 64, T, R, 4, 2, 0.0, "hgt", True, True, True).to(dev).train()
    head = torch.nn.Linear(64, 5).to(dev)

    def fwd(x, nt, tm, ei, et):
        with torch.autocast("cuda", dtype=BF16):
            return gnn(x, nt, tm, ei, et)

    def loss_fn(x, nt, tm, ei, et, targets):
        with torch.autocast("cuda", dtype=BF16):
            h = gnn(x, nt, tm, ei, et)[:counts[0]]
            return F.nll_loss(F.log_softmax(head(h).float(), -1), targets[0], ignore_index=-100)

    gf = graphed.GraphedForward(fwd, sig, dev)
    params = list(gnn.parameters()) + list(head.parameters())
    step = graphed.GraphedTrainStep(loss_fn, sig, dev, params=params, targets={0: ((), torch.int64, -100)})
    with _deterministic(True), torch.no_grad():
        for b in batches * 2:
            x = torch.randn(b.num_nodes, F_IN, generator=torch.Generator().manual_seed(b.num_nodes))
            gf(x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
            torch.cuda.synchronize()
            got = gf.out.clone()
            gf._rebuild_plan()
            ref = fwd(gf.x, gf.nt, gf.tm, gf.ei, gf.et)
            assert torch.equal(got, ref)
    with _deterministic(True):
        for b in batches * 2:
            x = torch.randn(b.num_nodes, F_IN, generator=torch.Generator().manual_seed(7 + b.num_nodes))
            n0 = int((b.node_type == 0).sum())
            y = torch.randint(0, 5, (n0,), generator=torch.Generator().manual_seed(b.num_nodes))
            loss, = step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
            torch.cuda.synchronize()
            g_loss, g_grads = loss.clone(), [p.grad.clone() for p in params]
            static = [p.grad for p in params]
            for p in params:
                p.grad = None
            step._rebuild_plan()
            ref = step.loss_fn(step.x, step.nt, step.tm, step.ei, step.et, step.y)
            ref.backward()
            assert torch.equal(g_loss, ref.detach())
            for p, g_ in zip(params, g_grads):
                assert torch.equal(g_, p.grad)
            for p, g_ in zip(params, static):
                p.grad = g_
