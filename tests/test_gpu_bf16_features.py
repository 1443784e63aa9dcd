"""bf16 node features end to end: device-sampled bf16 batches, their merge and graphed copy-in, and the input adapter's
typed GEMM reading bf16 A (hgt_typed_linear_bf16a, hgt_typed_linear_bwd_bf16a[_det]).

A bf16 value is exactly the hi half of the split-bf16 scheme and its lo half is zero.  The bf16-A GEMMs skip the products
with that lo half, which only add exact zeros, and run the others in the fp32 path's order, so every result here is
compared BITWISE with the fp32 path fed the widened features (`x.float()`), and the GEMMs also against float64.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, graphed, plan as P          # noqa: E402
from tests.conftest import load_golden                   # noqa: E402
from tests.test_gpu_sampler import _gen, _tables         # noqa: E402
from tests.test_gpu_sampler_batched import _assert_bitwise, _inps   # noqa: E402
from tests.test_gpu_sampler_mask import _rules           # noqa: E402
from tests.test_sampler import _GraphStub                # noqa: E402

BF16 = torch.bfloat16
SENTINEL = -7.0


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


class _Det:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(self.on, warn_only=True)

    def __exit__(self, *a):
        torch.use_deterministic_algorithms(self.old)


class _Precision:
    def __init__(self, p):
        self.p = p

    def __enter__(self):
        self.old = torch.get_float32_matmul_precision()
        torch.set_float32_matmul_precision(self.p)

    def __exit__(self, *a):
        torch.set_float32_matmul_precision(self.old)


def _bits(t):
    return t.view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the typed GEMM with bf16 A: forward

def _table(width, ms, ncb):
    """Groups of m rows with `ncb` column blocks each, side by side in output rows of ld = ncb * width + 8."""
    groups, cblocks, a0, out0, w0 = [], [], 0, 0, 0
    ld = ncb * width + 8
    for g, m in enumerate(ms):
        groups.append((a0, m, w0, ncb, len(cblocks), g % 3 != 1))
        cblocks += [(out0 + cb * width, ld) for cb in range(ncb)]
        a0 += m
        out0 += m * ld
        w0 += ncb * width
    return P._pack_groups(groups, cblocks, _dev()), a0, out0, w0


def _operands(K, rows, w_rows, seed, lda=None):
    dev = _dev()
    gen = torch.Generator().manual_seed(seed)
    lda = K if lda is None else lda
    # the columns past K hold values that must not be read (NaN would poison a product that read them)
    a = (torch.randn(rows, lda, generator=gen) * 3).to(BF16)
    a[:, K:] = float("nan")
    a = a.to(dev)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    return a, w, b


def _fwd(fn, a, lda, w, b, K, width, tab, out_elems, impl):
    g_dev, g_host, n_g, c_dev = tab
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=a.device)
    out = torch.full((out_elems,), SENTINEL, dtype=torch.float32, device=a.device)
    _lib.call(fn, a.data_ptr(), lda, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g,
              c_dev.data_ptr(), out.data_ptr(), impl, ws.data_ptr(), ws.numel(), _st())
    return out


def _ref64(a, w, b, tab, width, ms, ncb, out_elems, K):
    """float64 output in the table's layout, and the error scale sum_k |a||w| per element."""
    g_host = tab[1]
    ld = ncb * width + 8
    ref = torch.full((out_elems,), SENTINEL, dtype=torch.float64)
    scale = torch.zeros(out_elems, dtype=torch.float64)
    a64, w64, b64 = a[:, :K].double().cpu(), w.double().cpu(), b.double().cpu()
    out0 = 0
    for g, m in enumerate(ms):
        a0, w0 = int(g_host["a_row0"][g]), int(g_host["w_row0"][g])
        for cb in range(ncb):
            ws = w64[w0 + cb * width:w0 + (cb + 1) * width]
            y = a64[a0:a0 + m] @ ws.T + (b64[w0 + cb * width:w0 + (cb + 1) * width] if g % 3 != 1 else 0)
            s = a64[a0:a0 + m].abs() @ ws.abs().T + 1.0
            idx = out0 + cb * width + torch.arange(m)[:, None] * ld + torch.arange(width)[None, :]
            ref[idx.reshape(-1)] = y.reshape(-1)
            scale[idx.reshape(-1)] = s.reshape(-1)
        out0 += m * ld
    return ref, scale


@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("width", [128, 400, 512])
@pytest.mark.parametrize("K", [64, 129, 256, 1169])
def test_forward_bf16a_equals_fp32_on_widened_a(K, width, impl):
    ms, ncb = (300, 77, 130), 2
    tab, rows, out_elems, w_rows = _table(width, ms, ncb)
    a, w, b = _operands(K, rows, w_rows, seed=K * 7 + width + impl)
    a32 = a.float().contiguous()
    got = _fwd("hgt_typed_linear_bf16a", a, K, w, b, K, width, tab, out_elems, impl)
    ref = _fwd("hgt_typed_linear", a32, K, w, b, K, width, tab, out_elems, impl)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(ref))
    r64, scale = _ref64(a, w, b, tab, width, ms, ncb, out_elems, K)
    tol = 8e-3 if impl == 3 else 2e-4                     # impl 3 rounds W to bf16 (A is exact)
    assert ((got.double().cpu() - r64).abs() <= tol * scale).all()


@pytest.mark.parametrize("impl", [2, 3])
@pytest.mark.parametrize("K,lda", [(256, 264), (256, 260), (129, 136)])
def test_forward_bf16a_strided_a(K, lda, impl):
    """A with a row stride past K: read in place (lda % 8 == 0, K % 8 == 0) or copied into padded rows first."""
    width, ms, ncb = 128, (200, 131), 1
    tab, rows, out_elems, w_rows = _table(width, ms, ncb)
    a, w, b = _operands(K, rows, w_rows, seed=lda + impl, lda=lda)
    a32 = a.float().contiguous()
    got = _fwd("hgt_typed_linear_bf16a", a, lda, w, b, K, width, tab, out_elems, impl)
    ref = _fwd("hgt_typed_linear", a32, lda, w, b, K, width, tab, out_elems, impl)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(ref))


# ---------------------------------------------------------------------------------------------------------------------
# 2. dW and db

def _bwd(a, K, width, tab, dout, w_rows, impl, det, bf16a, has_bias=True):
    dev = _dev()
    g_dev, g_host, n_g, _ = tab
    c_host = tab.c_host
    dw = torch.zeros(w_rows, K, device=dev)
    db = torch.zeros(w_rows, device=dev) if has_bias else None
    sfx = "_det" if det else ""
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_bwd" + sfx + "_workspace_bytes", g_host.ctypes.data, n_g, c_host.ctypes.data, K, width,
              K, dout.numel(), 0, int(bf16a), impl, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    if bf16a:
        _lib.call("hgt_typed_linear_bwd_bf16a" + sfx, dout.data_ptr(), dout.numel(), a.data_ptr(), K, K, width,
                  g_dev.data_ptr(), g_host.ctypes.data, n_g, c_host.ctypes.data, dw.data_ptr(), _lib.ptr(db), impl,
                  ws.data_ptr(), ws.numel(), _st())
    else:
        w = torch.zeros(w_rows, K, device=dev)               # the fp32 entry point wants W even without dA
        _lib.call("hgt_typed_linear_bwd" + sfx, dout.data_ptr(), None, None, dout.numel(), a.data_ptr(), K, None, None,
                  w.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data, n_g, c_host.ctypes.data, None, 0, None,
                  dw.data_ptr(), _lib.ptr(db), impl, ws.data_ptr(), ws.numel(), _st())
    return dw, db


# the tensor-core backward takes K % 16 == 0: the adapter runs K = 129 / 1169 on the SIMT kernels (impl 1)
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("width", [128, 400, 512])
@pytest.mark.parametrize("K,impl", [(64, 1), (64, 2), (64, 3), (129, 1), (256, 1), (256, 2), (256, 3), (1169, 1)])
def test_backward_bf16a_dw_db(K, impl, width, det):
    ms, ncb = (700, 333), 1
    tab, rows, out_elems, w_rows = _table(width, ms, ncb)
    a, _, _ = _operands(K, rows, w_rows, seed=K + width + impl)
    a = a.contiguous()
    dout = torch.randn(out_elems, generator=torch.Generator().manual_seed(K + 3 * width)).to(_dev())
    a32 = a.float().contiguous()
    dw, db = _bwd(a, K, width, tab, dout, w_rows, impl, det, True)
    rw, rb = _bwd(a32, K, width, tab, dout, w_rows, impl, det, False)
    torch.cuda.synchronize()
    if det:
        assert torch.equal(_bits(dw), _bits(rw)) and torch.equal(_bits(db), _bits(rb))
    # float64: dW[w0 + n, k] = sum_m dOut[m, n] a[a0 + m, k] over each group
    g_host = tab[1]
    ld = ncb * width + 8
    a64, d64 = a.double().cpu(), dout.double().cpu()
    out0 = 0
    tol = 8e-3 if impl == 3 else 2e-4
    for g, m in enumerate(ms):
        a0, w0 = int(g_host["a_row0"][g]), int(g_host["w_row0"][g])
        d = d64[out0:out0 + m * ld].view(m, ld)[:, :width]
        ref_w = d.T @ a64[a0:a0 + m]
        scale = d.abs().T @ a64[a0:a0 + m].abs() + 1.0
        assert ((dw[w0:w0 + width].double().cpu() - ref_w).abs() <= tol * scale).all()
        if g % 3 != 1:
            ref_b = d.sum(0)
            assert ((db[w0:w0 + width].double().cpu() - ref_b).abs() <= 1e-4 * (d.abs().sum(0) + 1.0)).all()
        out0 += m * ld


# ---------------------------------------------------------------------------------------------------------------------
# 3. sampler, merge

_GRAPHS = {}


def _bf16_graph(placement, width):
    from pyhgt_b200 import sampler
    key = (placement, width)
    if key not in _GRAPHS:
        fx = load_golden("sampler_large")
        g = _GraphStub(fx)
        fg = sampler.FrozenGraph(g)
        tabs = _tables(fg, g.get_types(), width=width, seed=width)
        _GRAPHS[key] = (fx, fg, sampler.DeviceGraph(fg, _dev(), tabs, placement=placement, feature_dtype=BF16))
    return _GRAPHS[key]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("placement", ["device", "host"])
@pytest.mark.parametrize("width", [128, 129, 1169, 37])
def test_bf16_batches_equal_fp32_batches(width, placement, masked):
    from pyhgt_b200 import sampler
    fx, fg, dg = _bf16_graph(placement, width)
    inps = _inps(fx, fg, 0, 5, seed=width)[:2] + [{"paper": np.array([[0, 2010], [1, 2011]])}]
    mask = _rules(16)["paper_field"] if masked else None
    a = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 16, inps, _gen(9), edge_mask=mask)
    b = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 16, inps, _gen(9), edge_mask=mask, feature_dtype=BF16)
    for x, y in zip(a, b):
        assert y[0].dtype == BF16 and y[0].shape == x[0].shape
        assert torch.equal(y[0].float(), x[0])
        _assert_bitwise((None,) + x[1:], (None,) + y[1:])
    one = sampler.sample_subgraph_cuda(dg, fx["time_range"], 3, 16, inps[0], _gen(9), feature_dtype=BF16)
    assert torch.equal(one[0], b[0][0])
    T, R = len(dg.types), len(dg.edge_dict)
    m32 = sampler.merge_batches(a, T, R)
    m16 = sampler.merge_batches(b, T, R)
    assert m16[0].dtype == BF16 and torch.equal(m16[0].float(), m32[0])
    for u, v in zip(m32[1:5], m16[1:5]):
        assert torch.equal(u, v)
    assert all(torch.equal(u, v) for u, v in zip(m32[5], m16[5]))


def test_bf16_batches_need_a_bf16_graph():
    from pyhgt_b200 import sampler
    from tests.test_gpu_sampler import _device_graph
    fx, _, _, dg32, _ = _device_graph("sampler")
    with pytest.raises(ValueError, match="feature_dtype"):
        sampler.sample_subgraph_cuda(dg32, fx["time_range"], 2, 8, fx["inp"], _gen(1), feature_dtype=BF16)
    with pytest.raises(ValueError, match="feature_dtype"):
        sampler.sample_subgraph_cuda(dg32, fx["time_range"], 2, 8, fx["inp"], _gen(1), feature_dtype=torch.float16)
    b32 = sampler.sample_subgraph_cuda(dg32, fx["time_range"], 2, 8, fx["inp"], _gen(1))
    b16 = (b32[0].to(BF16),) + tuple(b32[1:])
    with pytest.raises(ValueError, match="same dtype"):
        sampler.merge_batches([b32, b16], len(dg32.types), len(dg32.edge_dict))


# ---------------------------------------------------------------------------------------------------------------------
# 4. GNN: full and trimmed forwards, training

N_HID, N_CLS = 64, 5


def _paper_inps(fx, fg, B, seed):
    """The fixture's seeds, then B - 1 dicts of 16 other paper seeds."""
    rng = np.random.RandomState(seed)
    inps = [fx["inp"]]
    for _ in range(B - 1):
        ids = rng.choice(fg.n_ids["paper"], 16, replace=False)
        inps.append({"paper": np.stack([ids, rng.randint(2000, 2016, 16)], 1)})
    return inps


def _gnn_batch(width, B=3):
    from pyhgt_b200 import sampler
    fx, fg, dg = _bf16_graph("device", width)
    inps = _paper_inps(fx, fg, B, seed=width + 1)
    mem = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 16, inps, _gen(5), feature_dtype=BF16)
    T, R = len(dg.types), len(dg.edge_dict)
    x16, nt, tm, ei, et, _ = sampler.merge_batches(mem, T, R)
    return dg, (x16, nt, tm, ei, et), mem


def _model(dg, width, seed=3, dropout=0.0):
    from pyhgt_b200.model import GNN
    torch.manual_seed(seed)
    return GNN(width, N_HID, len(dg.types), len(dg.edge_dict), 4, 2, dropout, "hgt", True, False, True).to(_dev())


@pytest.mark.parametrize("precision", ["highest", "medium"])
@pytest.mark.parametrize("width", [129, 1169])
def test_gnn_forwards_on_bf16_equal_widened(width, precision):
    from pyhgt_b200 import trim
    dg, (x16, nt, tm, ei, et), mem = _gnn_batch(width)
    gnn = _model(dg, width).eval()
    paper = dg.slot["paper"]
    T, R = len(dg.types), len(dg.edge_dict)
    x32 = x16.float()
    with _Precision(precision), torch.no_grad():
        assert torch.equal(gnn(x16, nt, tm, ei, et), gnn(x32, nt, tm, ei, et))
        rows = torch.nonzero(nt == paper).view(-1)[:20].contiguous()
        assert torch.equal(gnn(x16, nt, tm, ei, et, out_nodes=rows), gnn(x32, nt, tm, ei, et, out_nodes=rows))
        tsig = trim.TrimSignature.for_batches([(x16, nt, tm, ei, et)], [rows], 2, 0.1, num_types=T, num_relations=R)
        assert torch.equal(gnn(x16, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig),
                           gnn(x32, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig))
        # an unsorted node order (not what to_torch emits): the rows are gathered with index_select
        perm = torch.randperm(nt.numel(), generator=torch.Generator().manual_seed(0)).to(nt.device)
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(perm.numel(), device=perm.device)
        ei_p = inv[ei]
        assert torch.equal(gnn(x16[perm], nt[perm], tm, ei_p, et), gnn(x32[perm], nt[perm], tm, ei_p, et))


@pytest.mark.parametrize("trimmed", [False, True])
@pytest.mark.parametrize("precision", ["highest", "medium"])
@pytest.mark.parametrize("width", [129, 1169, 256])          # 256: the adapter's tensor-core forward and dW
def test_gnn_training_on_bf16_equals_widened(width, precision, trimmed):
    dg, (x16, nt, tm, ei, et), mem = _gnn_batch(width)
    paper = dg.slot["paper"]
    rows = torch.nonzero(nt == paper).view(-1)[:24].contiguous()
    y = torch.randint(0, N_CLS, (rows.numel(),), generator=torch.Generator().manual_seed(1)).to(_dev())
    res = []
    for x in (x16, x16.float()):
        gnn = _model(dg, width).train()
        head = torch.nn.Linear(N_HID, N_CLS).to(_dev())
        torch.manual_seed(0)
        with _Precision(precision), _Det(True):
            h = gnn(x, nt, tm, ei, et, out_nodes=rows) if trimmed else gnn(x, nt, tm, ei, et)[rows]
            loss = F.nll_loss(F.log_softmax(head(h), -1), y)
            loss.backward()
        torch.cuda.synchronize()
        res.append((loss.detach(), [p.grad.clone() for p in list(gnn.parameters()) + list(head.parameters())]))
    (l16, g16), (l32, g32) = res
    assert torch.equal(l16, l32)
    assert len(g16) == len(g32) and all(torch.equal(a, b) for a, b in zip(g16, g32))


def test_gnn_dtype_errors():
    dg, (x16, nt, tm, ei, et), _ = _gnn_batch(129, B=1)
    gnn = _model(dg, 129)
    for dt in (torch.float16, torch.float64):
        with pytest.raises(ValueError, match="float32 or bfloat16"):
            gnn(x16.to(dt), nt, tm, ei, et)
        with torch.no_grad(), pytest.raises(ValueError, match="float32 or bfloat16"):
            gnn(x16.to(dt), nt, tm, ei, et, out_nodes=torch.zeros(1, dtype=torch.int64, device=_dev()))
    with pytest.raises(ValueError, match="require grad"):
        gnn(x16.clone().requires_grad_(True), nt, tm, ei, et)


# ---------------------------------------------------------------------------------------------------------------------
# 5. graphed classes

def test_graphed_classes_with_a_bf16_signature():
    from pyhgt_b200 import sampler
    width = 129
    fx, fg, dg = _bf16_graph("device", width)
    inps = _paper_inps(fx, fg, 4, seed=11)
    members = sampler.sample_subgraphs_cuda(dg, fx["time_range"], 3, 8, inps, _gen(3), feature_dtype=BF16)
    T, R = len(dg.types), len(dg.edge_dict)
    plans = [P.get_plan(m[1], m[3], m[4], m[2], T, R) for m in members]
    counts = [max(p.type_count[t] for p in plans) + 3 for t in range(T)]
    pairs = {pr for p in plans for pr in p.pairs}
    E = max(p.n_edges for p in plans) + 50
    sig16 = graphed.GraphSignature(counts, E, pairs, R, width, feat_dtype=BF16)
    sig32 = graphed.GraphSignature(counts, E, pairs, R, width)
    paper = dg.slot["paper"]
    r0, C = int(sig16.row0[paper]), sig16.type_counts[paper]
    labels = [torch.randint(0, N_CLS, (p.type_count[paper],), generator=torch.Generator().manual_seed(b)).to(_dev())
              for b, p in enumerate(plans)]
    outs = {}
    for sig in (sig16, sig32):
        gnn = _model(dg, width)
        head = torch.nn.Linear(N_HID, N_CLS).to(_dev())
        params = list(gnn.parameters()) + list(head.parameters())

        def loss_fn(x, nt, tm, ei, et, targets, gnn=gnn, head=head):
            h = gnn(x, nt, tm, ei, et)[r0:r0 + C]
            return F.nll_loss(F.log_softmax(head(h), -1), targets[paper], ignore_index=-100)

        fwd = graphed.GraphedForward(lambda x, nt, tm, ei, et, gnn=gnn: gnn(x, nt, tm, ei, et), sig, _dev())
        step = graphed.GraphedTrainStep(loss_fn, sig, _dev(), params=params, targets={paper: ((), torch.int64, -100)})
        got = []
        with _Det(True):
            for rep in range(2):
                for b, m in enumerate(members):
                    nf = m[0] if sig is sig16 else m[0].float()
                    gnn.eval()
                    out = fwd(nf, *m[1:5]).clone()
                    gnn.train()
                    loss, = step(nf, *m[1:5], targets={paper: labels[b]})
                    torch.cuda.synchronize()
                    got.append((out, loss.clone(), [p.grad.clone() for p in params]))
        # a host batch takes the same padding path (16-bit patterns for bf16)
        host = tuple(t.cpu() for t in members[0][:5])
        if sig is sig32:
            host = (host[0].float(),) + host[1:]
        gnn.eval()
        got.append((fwd(*host).clone(), None, None))
        outs[sig is sig16] = got
    for (o16, l16, g16), (o32, l32, g32) in zip(outs[True], outs[False]):
        assert torch.equal(o16, o32)
        if l16 is not None:
            assert torch.equal(l16, l32) and all(torch.equal(a, b) for a, b in zip(g16, g32))
    # a batch whose dtype is not the signature's
    m = members[0]
    fwd16 = graphed.GraphedForward(lambda *a: a[0], sig16, _dev())
    with pytest.raises(ValueError, match="node_feature"):
        fwd16(m[0].float(), *m[1:5])
    with pytest.raises(ValueError, match="feat_dtype"):
        fwd16(m[0].float().cpu(), *(t.cpu() for t in m[1:5]))
