"""torch.set_float32_matmul_precision("medium"): the typed GEMMs run one bf16 product (C impl 3, or a presplit call with
a_lo == NULL) instead of the split-bf16 x3.

  kernels     the forward (BN 64 / 128 / 256, fp32 and bf16 output, tensor-store and staged epilogues, group tails, more
              than 64 groups) and the backward (dX with and without gelu', dW, atomic and deterministic) against float64
              on the bf16-rounded operands; the x3 path must be at least 10x farther from that reference, which is what
              shows that one product ran
  producers   every hi-only output equals the hi half of the hi/lo output, bitwise
  layers      HGTConv / GNN / DenseHGTConv against the reference fixtures, trimmed rows, graphs, determinism, and that
              "highest" / "high" are untouched by a "medium" run
"""
import contextlib
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, plan as P, synth          # noqa: E402
from tests.conftest import load_golden                 # noqa: E402

BF16 = torch.bfloat16
# Per-element bound of a one-product GEMM against float64 on the bf16-rounded operands: the products are exact in fp32,
# so only the fp32 accumulation remains.  ACC_TOL * (sum_k |a_k w_k| + |b|).
ACC_TOL = 1e-5
# Layer outputs at "medium" against the reference fixtures (LayerNorm'd outputs: max-abs, relative Frobenius) and
# gradients (relative Frobenius).  DESIGN.md §5.2 records the measured values.
OUT_MAX_ABS, OUT_REL_FRO, GRAD_REL_FRO = 5e-2, 1e-2, 2e-2


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30))


@contextlib.contextmanager
def _precision(p):
    old = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision(p)
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(old)


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _rne(t):
    """float64 copy of t rounded to bf16 (nearest-even), on the host."""
    return t.detach().to(BF16).double().cpu()


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward kernel

def _table(width, ms, ncb, pad):
    groups, cblocks, a0, out0, w0 = [], [], 0, 0, 0
    ld = ncb * width + pad
    for g, m in enumerate(ms):
        groups.append((a0, m, w0, ncb, len(cblocks), g % 3 != 1))
        cblocks += [(out0 + cb * width, ld) for cb in range(ncb)]
        a0 += m
        out0 += m * ld
        w0 += ncb * width
    return P._pack_groups(groups, cblocks, _dev()), a0, out0, w0


def _ref_fwd(tab, width, a, w, b, out_elems):
    """float64 out and the bound's scale sum_k |a_k w_k| + |b| over the covered elements (idx)."""
    g_host, n_g, c_host = tab[1], tab[2], tab.c_host
    ref = torch.zeros(out_elems, dtype=torch.float64)
    scale = torch.zeros(out_elems, dtype=torch.float64)
    idx = []
    for g in range(n_g):
        a0, m, w0, ncb, cb0, has_b = [int(g_host[g][k]) for k in ("a_row0", "m", "w_row0", "n_cblocks", "cb_first",
                                                                   "has_bias")]
        for cb in range(ncb):
            off, ld = int(c_host[cb0 + cb]["out_off"]), int(c_host[cb0 + cb]["ld"])
            ws = w[w0 + cb * width:w0 + (cb + 1) * width]
            bb = b[w0 + cb * width:w0 + (cb + 1) * width] if has_b else torch.zeros(width, dtype=torch.float64)
            i = (off + torch.arange(m)[:, None] * ld + torch.arange(width)[None]).reshape(-1)
            ref[i] = (a[a0:a0 + m] @ ws.T + bb).reshape(-1)
            scale[i] = (a[a0:a0 + m].abs() @ ws.abs().T + bb.abs()).reshape(-1)
            idx.append(i)
    return ref, scale, torch.cat(idx)


FWD_CASES = [
    # K, width, group rows, column blocks, ld pad
    (96, 64, [200, 37, 128], 2, 0),                    # BN = 64, staged epilogue
    (128, 128, [300, 129, 1], 2, 0),                   # BN = 128, tensor stores, tails of 1 / 44 rows
    (256, 256, [150, 257, 64], 2, 0),                  # BN = 256, tensor stores
    (256, 256, [150, 257], 1, 1),                      # BN = 256, unaligned ld: staged epilogue
    (128, 128, [190, 65], 2, 1),                       # BN = 128, unaligned ld
    (64, 400, [333, 64], 1, 0),                        # d = 400: BN = 64
    (64, 128, [17 + 5 * i for i in range(70)], 1, 0),  # more than 64 groups: chunked launches
]


@pytest.mark.parametrize("K,width,ms,ncb,pad", FWD_CASES)
def test_forward_one_product_matches_fp64(K, width, ms, ncb, pad):
    dev = _dev()
    tab, rows, out_elems, w_rows = _table(width, ms, ncb, pad)
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator().manual_seed(K + width + len(ms) + pad)
    a = (torch.randn(rows, K, generator=gen) * 2).to(dev)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    outs = {}
    for impl, dtype in ((3, torch.float32), (3, BF16), (2, torch.float32)):
        out = torch.zeros(out_elems, dtype=dtype, device=dev)
        wsb = ctypes.c_size_t()
        _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        _lib.call("hgt_typed_linear_bf16" if dtype == BF16 else "hgt_typed_linear", a.data_ptr(), K, w.data_ptr(),
                  b.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), out.data_ptr(),
                  impl, ws.data_ptr(), ws.numel(), _st())
        outs[(impl, dtype)] = out
    # the presplit entry point with a_lo == NULL: the same kernel on the same hi half
    hi = torch.empty(rows, K, dtype=BF16, device=dev)
    _lib.call("hgt_act_split", a.data_ptr(), K, rows, K, 0, None, hi.data_ptr(), None, _st())
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    pre = torch.zeros(out_elems, device=dev)
    _lib.call("hgt_typed_linear_presplit", hi.data_ptr(), None, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), pre.data_ptr(), ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()

    ref, scale, idx = _ref_fwd(tab, width, _rne(a), _rne(w), b.double().cpu(), out_elems)
    one = outs[(3, torch.float32)]
    err1 = (one.double().cpu() - ref)[idx]
    ratio = float((err1.abs() / scale[idx]).max())
    assert ratio <= ACC_TOL, "one product: max |err| / (sum |a w| + |b|) = %.3g" % ratio
    err3 = (outs[(2, torch.float32)].double().cpu() - ref)[idx]
    assert float(err3.norm()) >= 10 * float(err1.norm()), \
        "x3 is only %.3g x farther from the bf16-operand reference" % (float(err3.norm()) / float(err1.norm()))
    assert torch.equal(outs[(3, BF16)].view(torch.int16), one.to(BF16).view(torch.int16))
    assert torch.equal(pre, one)


# ---------------------------------------------------------------------------------------------------------------------
# 2. backward kernels

BWD_CASES = [
    # K (= dX tile width), width, group rows, column blocks
    (64, 128, [700, 300], 2),
    (128, 64, [600, 450, 37], 2),
    (256, 128, [520, 300, 100], 1),
]


def _bwd(fn, dout, d_hi, A, a_hi, W, K, width, tab, out_elems, gelu_aux, want_db, impl):
    dev = _dev()
    g_dev, g_host, n_g, _ = tab
    rows = A.shape[0]
    dA = torch.empty(rows, K, device=dev)
    dW = torch.zeros_like(W)
    db = torch.zeros(W.shape[0], device=dev) if want_db else None
    wsb = ctypes.c_size_t()
    _lib.call(fn + "_workspace_bytes", g_host.ctypes.data, n_g, tab.c_host.ctypes.data, K, width, K, out_elems,
              int(d_hi is not None), int(a_hi is not None), impl, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    _lib.call(fn, _lib.ptr(dout), _lib.ptr(d_hi), None, out_elems, A.data_ptr(), K, _lib.ptr(a_hi), None, W.data_ptr(),
              K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g, tab.c_host.ctypes.data, dA.data_ptr(), 0,
              _lib.ptr(gelu_aux), dW.data_ptr(), _lib.ptr(db), impl, ws.data_ptr(), ws.numel(), _st())
    return dA, dW, db


def _gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("K,width,ms,ncb", BWD_CASES)
def test_backward_one_product_matches_fp64(K, width, ms, ncb, gelu, det):
    dev = _dev()
    tab, rows, out_elems, w_rows = _table(width, ms, ncb, 0)
    gen = torch.Generator().manual_seed(K * 7 + width + int(gelu))
    dout = torch.randn(out_elems, generator=gen).to(dev)
    A = torch.randn(rows, K, generator=gen).to(dev)
    W = torch.randn(w_rows, K, generator=gen).to(dev)
    aux = torch.randn(rows, K, generator=gen).to(dev) if gelu else None
    fn = "hgt_typed_linear_bwd_det" if det else "hgt_typed_linear_bwd"
    dA, dW, db = _bwd(fn, dout, None, A, None, W, K, width, tab, out_elems, aux, True, 3)
    dA3, dW3, _ = _bwd(fn, dout, None, A, None, W, K, width, tab, out_elems, aux, True, 2)
    if det:
        again = _bwd(fn, dout, None, A, None, W, K, width, tab, out_elems, aux, True, 3)
        assert all(torch.equal(x, y) for x, y in zip((dA, dW, db), again))
        # operands pre-split by their producers, hi halves only: the same result bitwise (db is then not computed)
        d_hi = torch.empty(out_elems, dtype=BF16, device=dev)
        a_hi = torch.empty(rows, K, dtype=BF16, device=dev)
        _lib.call("hgt_act_split", dout.data_ptr(), out_elems, 1, out_elems, 0, None, d_hi.data_ptr(), None, _st())
        _lib.call("hgt_act_split", A.data_ptr(), K, rows, K, 0, None, a_hi.data_ptr(), None, _st())
        pre = _bwd(fn, None, d_hi, A, a_hi, W, K, width, tab, out_elems, aux, False, 3)
        assert torch.equal(pre[0], dA) and torch.equal(pre[1], dW)
    torch.cuda.synchronize()

    d_r, a_r, w_r = _rne(dout), _rne(A), _rne(W)
    ref_dA = torch.zeros(rows, K, dtype=torch.float64)
    sc_dA = torch.zeros(rows, K, dtype=torch.float64)
    ref_dW = torch.zeros(w_rows, K, dtype=torch.float64)
    sc_dW = torch.zeros(w_rows, K, dtype=torch.float64)
    ref_db = torch.zeros(w_rows, dtype=torch.float64)
    d64 = dout.double().cpu()
    g_host, c_host = tab[1], tab.c_host
    for g in range(tab[2]):
        a0, m, w0, n_cb, cb0, has_b = [int(g_host[g][k]) for k in ("a_row0", "m", "w_row0", "n_cblocks", "cb_first",
                                                                    "has_bias")]
        for cb in range(n_cb):
            off, ld = int(c_host[cb0 + cb]["out_off"]), int(c_host[cb0 + cb]["ld"])
            i = off + torch.arange(m)[:, None] * ld + torch.arange(width)[None]
            dd, ws = d_r[i], w_r[w0 + cb * width:w0 + (cb + 1) * width]
            ref_dA[a0:a0 + m] += dd @ ws
            sc_dA[a0:a0 + m] += dd.abs() @ ws.abs()
            ref_dW[w0 + cb * width:w0 + (cb + 1) * width] += dd.T @ a_r[a0:a0 + m]
            sc_dW[w0 + cb * width:w0 + (cb + 1) * width] += dd.abs().T @ a_r[a0:a0 + m].abs()
            if has_b:
                ref_db[w0 + cb * width:w0 + (cb + 1) * width] += d64[i].sum(0)
    bound_dA = ACC_TOL * sc_dA
    if gelu:
        # gelu'(aux) is evaluated in fp32 (erff, __expf): an absolute error of ~1e-6 on a factor that crosses zero
        gg = _gelu_grad(aux.double().cpu())
        ref_dA, bound_dA = ref_dA * gg, ACC_TOL * sc_dA * gg.abs() + 1e-6 * sc_dA
    tiny = 1e-30
    for got, ref, bound, x3, what in ((dA, ref_dA, bound_dA, dA3, "dX"), (dW, ref_dW, ACC_TOL * sc_dW, dW3, "dW")):
        err = got.double().cpu() - ref
        ratio = float((err.abs() / (bound + tiny)).max())
        assert ratio <= 1.0, "%s: max |err| / bound = %.3g" % (what, ratio)
        err3 = x3.double().cpu() - ref
        assert float(err3.norm()) >= 10 * float(err.norm()), "%s: x3 only %.3g x farther" % (
            what, float(err3.norm()) / float(err.norm()))
    torch.testing.assert_close(db.double().cpu(), ref_db, rtol=1e-5, atol=1e-4)


# ---------------------------------------------------------------------------------------------------------------------
# 3. hi-only producers

@pytest.mark.parametrize("act", [0, 1])
def test_act_split_hi_only(act):
    dev = _dev()
    x = torch.randn(777, 136, generator=torch.Generator().manual_seed(act)).to(dev)
    hi, lo, hi1 = (torch.full((777, 136), 7.0, dtype=BF16, device=dev) for _ in range(3))
    _lib.call("hgt_act_split", x.data_ptr(), 136, 777, 136, act, None, hi.data_ptr(), lo.data_ptr(), _st())
    _lib.call("hgt_act_split", x.data_ptr(), 136, 777, 136, act, None, hi1.data_ptr(), None, _st())
    torch.cuda.synchronize()
    assert torch.equal(hi.view(torch.int16), hi1.view(torch.int16))


@pytest.mark.parametrize("d,norm", [(64, True), (256, True), (400, False), (1024, True)])
def test_update_epilogue_hi_only(d, norm):
    dev = _dev()
    T, N = 3, 1000
    gen = torch.Generator().manual_seed(d)
    o, x = torch.randn(N, d, generator=gen).to(dev), torch.randn(N, d, generator=gen).to(dev)
    row0 = torch.tensor([0, 300, 710, N, N], dtype=torch.int32, device=dev)
    skip = torch.randn(T, generator=gen).to(dev)
    nw = torch.randn(T, d, generator=gen).to(dev) if norm else None
    nb = torch.randn(T, d, generator=gen).to(dev) if norm else None
    res = []
    for pair in (True, False):
        out = torch.empty(N, d, device=dev)
        hi = torch.full((N, d), 7.0, dtype=BF16, device=dev)
        lo = torch.full((N, d), 7.0, dtype=BF16, device=dev) if pair else None
        _lib.call("hgt_update_epilogue", o.data_ptr(), x.data_ptr(), row0.data_ptr(), T, skip.data_ptr(),
                  _lib.ptr(nw), _lib.ptr(nb), None, None, N, d, out.data_ptr(), hi.data_ptr(), _lib.ptr(lo), _st())
        res.append((out, hi))
    torch.cuda.synchronize()
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1].view(torch.int16), res[1][1].view(torch.int16))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("d,H,rte", [(64, 4, False), (256, 8, True), (128, 1, False), (512, 8, True)])
def test_edge_forward_hi_only(d, H, rte, variant, dtype):
    from tests.test_gpu_edge_instances import _plan, _tables
    dev = _dev()
    plan, T = _plan(d, H, rte, seed=d + H)
    q, kv, kvr = _tables(plan, d, rte, d, torch.float32 if dtype == "fp32" else BF16)
    N, E = plan.n_nodes, plan.n_edges
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    his = []
    for pair in (True, False):
        hi = torch.full((N, d), 7.0, dtype=BF16, device=dev)
        lo = torch.full((N, d), 7.0, dtype=BF16, device=dev) if pair else None
        _lib.call("hgt_edge_forward" + ("_bf16" if dtype == "bf16" else ""), q.data_ptr(), kv.data_ptr(),
                  _lib.ptr(kvr), plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
                  plan.rte_row.data_ptr() if rte else None, plan.csr_eid.data_ptr(), plan.tiles.data_ptr(),
                  plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, N, E, d, H, 1, None, None, None,
                  hi.data_ptr(), _lib.ptr(lo), ws.data_ptr(), ws.numel(), variant, _lib.ptr(plan.tile_counts_dev),
                  plan.type_row0_dev.data_ptr(), T, None, _st())
        his.append(hi)
    torch.cuda.synchronize()
    assert torch.equal(his[0].view(torch.int16), his[1].view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# 4. layers

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


def _close(got, ref, what):
    assert got.dtype == torch.float32 and torch.isfinite(got).all(), what
    err, fro = float((got.cpu() - ref.cpu()).abs().max()), _rel(got, ref)
    assert err <= OUT_MAX_ABS and fro <= OUT_REL_FRO, "%s: max-abs %.3g, rel-Frobenius %.3g" % (what, err, fro)


@pytest.mark.parametrize("fused", [True, False])
def test_conv_fixture_at_medium(conv_fixture, fused):
    fx, dev = conv_fixture, _dev()
    m = _conv(fx, dev)
    m.fused_call = fused
    args = _inputs(fx, dev)
    with torch.no_grad():
        hi = m(*args)
        with _precision("medium"):
            out = m(*args)
        again = m(*args)
    _close(out, fx["out"], "%s at medium (fused %s)" % (fx["name"], fused))
    assert torch.equal(hi, again)                        # "highest" after "medium" equals "highest" before
    if fx["cfg"]["out_dim"] >= 64 and fx["cfg"]["out_dim"] % 16 == 0:
        assert not torch.equal(out, hi)                  # the tensor-core GEMMs did change


def test_conv_d256_h8_at_medium():
    import pyhgt_b200
    dev = _dev()
    g = synth.make_random(3000, 30000, 3, 4, seed=5, self_loops=20)
    torch.manual_seed(1)
    m = pyhgt_b200.HGTConv(256, 256, 3, 4, 8, 0.0, True, True).to(dev).eval()
    x = torch.randn(3000, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    args = (x, g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    with torch.no_grad():
        ref = m(*args)
        for fused in (True, False):
            m.fused_call = fused
            with _precision("medium"):
                out = m(*args)
            _close(out, ref, "d256 H8 at medium vs highest (fused %s)" % fused)
        m.fused_call = True


def _grad_check(got, ref, what):
    assert got is not None, "no gradient for " + what
    fro = _rel(got, ref)
    assert fro <= GRAD_REL_FRO, "%s: relative Frobenius %.3g" % (what, fro)


def test_gnn_gradients_at_medium():
    from pyhgt_b200.model import GNN
    dev = _dev()
    fx = load_golden("gnn_2layer")
    c = fx["cfg"]
    m = GNN(c["in_dim"], c["n_hid"], c["num_types"], c["num_relations"], c["n_heads"], c["n_layers"], 0.2, "hgt",
            c["prev_norm"], c["last_norm"], c["use_RTE"])
    m.load_state_dict(fx["state_dict"], strict=True)
    m = m.to(dev).eval()
    x = fx["node_feature"].to(dev).requires_grad_(True)
    with _precision("medium"):
        out = m(x, fx["node_type"].to(dev), fx["edge_time"].to(dev), fx["edge_index"].to(dev), fx["edge_type"].to(dev))
        (out * fx["grad_weight"].to(dev)).sum().backward()
    _close(out.detach(), fx["out"], "GNN out at medium")
    _grad_check(x.grad, fx["grad_node_feature"], "d node_feature")
    got = dict(m.named_parameters())
    for k, ref in fx["grad_params"].items():
        _grad_check(got[k].grad, ref, "d " + k)


def test_dense_hgt_gradients_at_medium():
    import pyhgt_b200
    dev = _dev()
    fx = load_golden("dense_hgt")
    c = fx["cfg"]
    g = pyhgt_b200.GeneralConv('dense_hgt', c["in_dim"], c["out_dim"], c["num_types"], c["num_relations"], c["n_heads"],
                               0.2, c["use_norm"], c["use_RTE"])
    g.base_conv.load_state_dict(fx["state_dict"], strict=True)
    g = g.to(dev).eval()
    x = fx["node_inp"].to(dev).requires_grad_(True)
    with _precision("medium"):
        out = g(x, fx["node_type"].to(dev), fx["edge_index"].to(dev), fx["edge_type"].to(dev), fx["edge_time"].to(dev))
        (out * fx["grad_weight"].to(dev)).sum().backward()
    _close(out.detach(), fx["out"], "dense_hgt out at medium")
    _grad_check(x.grad, fx["grad_node_inp"], "d node_inp")
    got = dict(g.base_conv.named_parameters())
    for k, ref in fx["grad_params"].items():
        _grad_check(got[k].grad, ref, "d " + k)


def _gnn_setup(dev, kind="hgt", seed=4):
    from pyhgt_b200.model import GNN
    T, R = 3, 4
    g = synth.make_random(700, 5000, T, R, seed=seed, self_loops=20)
    x = torch.randn(700, 96, generator=torch.Generator().manual_seed(1)).to(dev)
    args = (g.node_type.to(dev), g.edge_time.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
    torch.manual_seed(0)
    gnn = GNN(96, 64, T, R, 4, 3, 0.0, kind, True, True, True).to(dev)
    return gnn, x, args


def _train_grads(gnn, x, args):
    gnn.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    y = gnn(xg, *args)
    y.square().mean().backward()
    return [y.detach(), xg.grad] + [p.grad.clone() for p in gnn.parameters()]


@pytest.mark.parametrize("kind", ["hgt", "dense_hgt"])
def test_nothing_leaks_between_settings(kind):
    """"highest" and "high" give bitwise equal outputs and gradients, before and after a "medium" run in the same
    process (plan / layer-table caches, split hints, workspaces)."""
    dev = _dev()
    gnn, x, args = _gnn_setup(dev, kind)
    with _deterministic(True):
        with torch.no_grad():
            inf0 = gnn.eval()(x, *args)
        gnn.train()
        first = _train_grads(gnn, x, args)
        with _precision("high"):
            high = _train_grads(gnn, x, args)
        with _precision("medium"):
            med = _train_grads(gnn, x, args)
            with torch.no_grad():
                inf_med = gnn.eval()(x, *args)
            gnn.train()
        after = _train_grads(gnn, x, args)
        with torch.no_grad():
            inf1 = gnn.eval()(x, *args)
    for a, b, c in zip(first, high, after):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert torch.equal(inf0, inf1)
    assert not torch.equal(med[0], first[0]) and not torch.equal(inf_med, inf0)
    assert _rel(med[0], first[0]) <= OUT_REL_FRO and _rel(inf_med, inf0) <= OUT_REL_FRO


def test_deterministic_training_at_medium():
    dev = _dev()
    gnn, x, args = _gnn_setup(dev)
    gnn.train()
    with _deterministic(True), _precision("medium"):
        a = _train_grads(gnn, x, args)
        b = _train_grads(gnn, x, args)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_trimmed_rows_equal_full_forward_at_medium():
    dev = _dev()
    gnn, x, args = _gnn_setup(dev)
    gnn.eval()
    out_nodes = torch.tensor([3, 10, 10, 250, 699, 0, 512], device=dev)
    with torch.no_grad(), _precision("medium"):
        full = gnn(x, *args)
        trimmed = gnn(x, *args, out_nodes=out_nodes)
    assert torch.equal(trimmed, full[out_nodes])


def test_sync_free_batch_at_medium():
    import pyhgt_b200
    from pyhgt_b200 import data as hdata
    from tests.test_data_ingest import _GraphStub
    dev = _dev()
    fx = load_golden("to_torch")
    g = _GraphStub(fx["types"], fx["meta_graph"])
    T = len(fx["types"])

    def batch():
        nf, nt, etime, ei, et, node_dict, edge_dict = hdata.to_torch(fx["feature"], fx["time"], fx["edge_list"], g,
                                                                    device=dev, prebuild_plan=True)
        return nf, nt, etime, ei, et, len(edge_dict)

    nf, nt, etime, ei, et, R = batch()
    d = nf.shape[1]
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, T, R, 1, 0.0, True, False).to(dev).eval()
    with torch.no_grad(), _precision("medium"):
        ref = m(nf, nt, ei, et)
        torch.cuda.synchronize()
        P.clear_plan_cache()
        nf2, nt2, etime2, ei2, et2, _ = batch()         # the cached plan holds etime2 by weak reference
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = m(nf2, nt2, ei2, et2)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(ref, got)


def test_graphed_train_step_at_medium():
    from pyhgt_b200 import graphed
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R, F_IN = 3, 4, 64
    batches = [synth.make_random(n, e, T, R, seed=s, sorted_types=True, self_loops=20)
               for n, e, s in ((400, 3000, 1), (310, 2200, 2))]
    counts = [max(int((b.node_type == t).sum()) for b in batches) + 5 for t in range(T)]
    pairs = {(int(b.node_type[s_]), int(r_)) for b in batches
             for s_, r_ in zip(b.edge_index[0].tolist(), b.edge_type.tolist())}
    sig = graphed.GraphSignature(counts, max(b.edge_type.numel() for b in batches) + 100, pairs, R, F_IN)
    torch.manual_seed(11)
    gnn = GNN(F_IN, 64, T, R, 4, 2, 0.0, "hgt", True, True, True).to(dev).train()
    head = torch.nn.Linear(64, 5).to(dev)

    def loss_fn(x, nt, tm, ei, et, targets):
        h = gnn(x, nt, tm, ei, et)[:counts[0]]
        return F.nll_loss(F.log_softmax(head(h), -1), targets[0], ignore_index=-100)

    params = list(gnn.parameters()) + list(head.parameters())
    step = graphed.GraphedTrainStep(loss_fn, sig, dev, params=params, targets={0: ((), torch.int64, -100)})
    gf = graphed.GraphedForward(lambda x, nt, tm, ei, et: gnn(x, nt, tm, ei, et), sig, dev)
    with _deterministic(True), _precision("medium"):
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
        b = batches[0]
        x = torch.randn(b.num_nodes, F_IN, generator=torch.Generator().manual_seed(3))
        with torch.no_grad():
            gf(x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
    b = batches[0]
    y = torch.zeros(int((b.node_type == 0).sum()), dtype=torch.int64)
    with _deterministic(True):                           # only the precision setting differs from the capture
        with pytest.raises(ValueError, match="captured with one-product"):
            step(x, b.node_type, b.edge_time, b.edge_index, b.edge_type, targets={0: y})
        with pytest.raises(ValueError, match="captured with one-product"), torch.no_grad():
            gf(x, b.node_type, b.edge_time, b.edge_index, b.edge_type)
