"""Fused dropout on the GPU (HGTConv.fused_dropout / GNN.fused_dropout; contract: include/hgt_b200.h "Fused dropout").

  * the masks the kernels draw equal the numpy restatement of the contract (tests/test_fused_dropout_cpu.py) bit for
    bit, at every epilogue instance, with perm / type_active, and for the adapter's tanh kernel;
  * forward and both backward kernels against float64 with that mask as a fixed multiplier, every instance;
  * HGTConv against float64 autograd through the oracle port with the layer's masks injected; DenseHGTConv and a
    2-layer GNN against their own nn.Dropout path with the same masks injected in place of nn.Dropout's;
  * the switch is inert in eval(), at p = 0 and when off; seeds reproduce; the step holds less memory; a captured
    training step draws new masks per replay, freezes the switch, and still learns.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tests import test_gpu_small_stage_instances as S          # noqa: E402
from tests.test_fused_dropout_cpu import drop_mask, drop_scale  # noqa: E402
from tests.test_gpu_grad_parity import _compare_all, _f64_params, _graph, _native_layer, _perturb  # noqa: E402

SEED = 0x1234_5678_9ABC_DEF


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _seed_tensor(seed, dev):
    return torch.tensor([seed], dtype=torch.int64, device=dev)


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- the mask, recovered from the kernels ---------------------------------------------------------------------------
def _epilogue_mask(d, mode, p, dev):
    """hgt_update_epilogue_drop with o = 1, x = 0, residual mode, no norm: out = mask * s.  Returns (out [N, d] with NaN
    where nothing was written, (rank row, output row) pairs of the rows the epilogue writes, unknown-type row start)."""
    L = S._lib()
    row0 = S._row0(S.FWD_COUNTS, S.FWD_UNKNOWN)
    N, T = row0[-1], len(S.FWD_COUNTS)
    perm, active, _, misaligned = S._epilogue_case(d, mode, seed=d)
    buf = torch.ones(N * d + 4, device=dev)
    o = buf[1:1 + N * d].view(N, d) if misaligned else buf[:N * d].view(N, d)
    x = torch.zeros(N, d, device=dev)
    out = S._nan(N, d, dev=dev)
    tr0, seed = S._i32(row0, dev), _seed_tensor(SEED + d, dev)
    perm_d = S._i32(perm, dev) if perm is not None else None
    act_d = S._i32(active, dev) if active is not None else None
    L.call("hgt_update_epilogue_drop", o.data_ptr(), x.data_ptr(), tr0.data_ptr(), T, None, None, None, L.ptr(perm_d),
           L.ptr(act_d), N, d, out.data_ptr(), None, None, seed.data_ptr(), p, S._st())
    torch.cuda.synchronize()
    return out.cpu(), S._expected_rows(perm, active, N), row0[T]


@pytest.mark.parametrize("p", [0.2, 0.5, 1.0])
@pytest.mark.parametrize("mode", ["plain", "perm_active", "misaligned"])
@pytest.mark.parametrize("d", [64, 78, 256, 400, 1000])
def test_epilogue_mask_is_the_contract(d, mode, p):
    """Vector instances NV 1 / 2 / 4 / 8 (d = 64, 256, 400, 1000), the scalar kernel (d = 78, and every d misaligned):
    row `row` of the mask lands in output row perm[row], rows without an output draw nothing."""
    out, rows, n_known = _epilogue_mask(d, mode, p, _dev())
    N = out.shape[0]
    want = torch.from_numpy(drop_mask(SEED + d, N, d, p)).float() * float(drop_scale(p))
    written = torch.zeros(N, dtype=torch.bool)
    for src, dst in rows:
        written[dst] = True
        exp = want[src] if src < n_known else torch.zeros(d)          # unknown type: zeros, nothing drawn
        assert torch.equal(_bits(out[dst]), _bits(exp)), (d, mode, p, src)
    assert torch.isnan(out[~written]).all()


def test_kept_fraction():
    dev = _dev()
    L = S._lib()
    N, d = 8192, 256
    o, x, out = torch.ones(N, d, device=dev), torch.zeros(N, d, device=dev), torch.empty(N, d, device=dev)
    tr0, seed = S._i32([0, N, N], dev), _seed_tensor(77, dev)
    for p in (0.2, 0.5):
        L.call("hgt_update_epilogue_drop", o.data_ptr(), x.data_ptr(), tr0.data_ptr(), 1, None, None, None, None, None,
               N, d, out.data_ptr(), None, None, seed.data_ptr(), p, S._st())
        kept = float((out != 0).double().mean())
        se = (p * (1 - p) / (N * d)) ** 0.5
        assert abs(kept - (1 - p)) < 5 * se, (p, kept)


# ---- tanh + dropout of the adapter ----------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.2, 1.0])
@pytest.mark.parametrize("d,misaligned", [(64, False), (78, False), (256, True), (400, False)])
def test_tanh_dropout_pair(d, misaligned, p):
    """Mask bitwise the contract; out and d x against float64 with the mask as a fixed multiplier; rows past n_rows
    pass unchanged in both directions; in place equals out of place."""
    dev = _dev()
    L = S._lib()
    n_rows, N = 301, 310
    gen = torch.Generator().manual_seed(d)
    x, g = 1.5 * torch.randn(N, d, generator=gen), torch.randn(N, d, generator=gen)
    buf = torch.empty(N * d + 4, device=dev)
    x_d = buf[1:1 + N * d].view(N, d) if misaligned else buf[:N * d].view(N, d)
    x_d.copy_(x)
    seed = _seed_tensor(SEED ^ d, dev)
    out, d_x = S._nan(N, d, dev=dev), S._nan(N, d, dev=dev)
    L.call("hgt_tanh_dropout", x_d.data_ptr(), n_rows, N, d, seed.data_ptr(), p, out.data_ptr(), S._st())
    g_d = g.to(dev)
    L.call("hgt_tanh_dropout_bwd", g_d.data_ptr(), out.data_ptr(), n_rows, N, d, seed.data_ptr(), p, d_x.data_ptr(),
           S._st())
    inplace = x_d.clone()
    L.call("hgt_tanh_dropout", inplace.data_ptr(), n_rows, N, d, seed.data_ptr(), p, inplace.data_ptr(), S._st())
    torch.cuda.synchronize()
    out, d_x = out.cpu(), d_x.cpu()
    assert torch.equal(_bits(inplace.cpu()), _bits(out))
    mask = torch.from_numpy(drop_mask(SEED ^ d, n_rows, d, p))
    assert torch.equal(out[:n_rows] != 0, mask & (x[:n_rows] != 0))
    assert torch.equal(_bits(out[n_rows:]), _bits(x[n_rows:])) and torch.equal(_bits(d_x[n_rows:]), _bits(g[n_rows:]))
    x64 = x[:n_rows].double().requires_grad_(True)
    ref = torch.tanh(x64) * mask.double() * float(drop_scale(p))
    (ref * g[:n_rows].double()).sum().backward()
    assert S._scaled_max(out[:n_rows], ref.detach(), 1.0) < 5e-6
    assert S._scaled_max(d_x[:n_rows], x64.grad, 1.0) < 5e-6


# ---- epilogue forward and backward against float64 ------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["plain", "perm_active", "misaligned"])
@pytest.mark.parametrize("d", S.WIDTHS)
def test_update_epilogue_drop_matches_fp64(d, mode):
    """hgt_update_epilogue_drop at every instance against the float64 epilogue of o * mask * s, skip and LayerNorm on
    and off, with the bf16 split bitwise where it is legal; tolerances of test_update_epilogue_matches_fp64."""
    dev = _dev()
    L = S._lib()
    p = 0.2
    o, x, skip, nw, nb, bias = S._epilogue_inputs(d, seed=d)
    N, T = o.shape[0], len(S.FWD_COUNTS)
    row0 = S._row0(S.FWD_COUNTS, S.FWD_UNKNOWN)
    perm, active, _, misaligned = S._epilogue_case(d, mode, seed=d)
    rows = S._expected_rows(perm, active, N)
    src, dst_rows = torch.tensor([r for r, _ in rows]), torch.tensor([w for _, w in rows])
    mask = torch.from_numpy(drop_mask(SEED + d, N, d, p)).double() * float(drop_scale(p))
    # the mean-1e4 rows of the plain test lose their small variance under a mask: keep them out of the LayerNorm bound
    edge = torch.zeros(N, dtype=torch.bool)
    edge[row0[3]:row0[3] + S.N_BIG + S.N_CONST] = True
    buf = torch.empty(N * d + 4, device=dev)
    o_dev = buf[1:1 + N * d].view(N, d) if misaligned else buf[:N * d].view(N, d)
    o_dev.copy_(o)
    x_d, tr0, seed = x.to(dev), S._i32(row0, dev), _seed_tensor(SEED + d, dev)
    perm_d = S._i32(perm, dev) if perm is not None else None
    act_d = S._i32(active, dev) if active is not None else None
    split_ok = perm is None and active is None and d % 8 == 0 and not misaligned
    for use_skip in (True, False):
        for use_norm in (True, False):
            s = skip if use_skip else None
            w, b = (nw, nb) if use_norm else (None, None)
            ref = S._epilogue_ref((o.double() * mask), x, s, w, b, None, bias)
            out = S._nan(N, d, dev=dev)
            hi = torch.full((N, d), 7.0, dtype=torch.bfloat16, device=dev) if split_ok else None
            lo = torch.full((N, d), 7.0, dtype=torch.bfloat16, device=dev) if split_ok else None
            s_d, w_d, b_d = (t.to(dev) if t is not None else None for t in (s, w, b))
            L.call("hgt_update_epilogue_drop", o_dev.data_ptr(), x_d.data_ptr(), tr0.data_ptr(), T, L.ptr(s_d),
                   L.ptr(w_d), L.ptr(b_d), L.ptr(perm_d), L.ptr(act_d), N, d, out.data_ptr(), L.ptr(hi), L.ptr(lo),
                   seed.data_ptr(), p, S._st())
            torch.cuda.synchronize()
            out = out.cpu()
            what = "d=%d %s skip=%s norm=%s" % (d, mode, use_skip, use_norm)
            unwritten = torch.ones(N, dtype=torch.bool)
            unwritten[dst_rows] = False
            assert torch.isnan(out[unwritten]).all(), what
            ok = ~edge[src] if use_norm else torch.ones(len(src), dtype=torch.bool)
            got, exp = out[dst_rows].double()[ok], ref[src][ok]
            e = (S._scaled_max(got, exp), S._rel_fro(got, exp))
            assert e[0] < 5e-6 and e[1] < 2e-6, (what, e)
            assert torch.isfinite(out[dst_rows]).all(), what
            if split_ok:
                eh, el = S._bf16_split(out)
                assert torch.equal(hi.cpu().view(torch.int16), eh) and torch.equal(lo.cpu().view(torch.int16), el), what


def _run_drop_bwd(o, x, g, skip, nw, perm, active, det, seed, p, dev):
    L = S._lib()
    row0 = S._row0(S.BWD_COUNTS, S.BWD_UNKNOWN)
    N, T, d = row0[-1], len(S.BWD_COUNTS), o.shape[1]
    o_d = o.clone()
    if active is not None:
        for t in range(T):
            o_d[row0[t] + active[t]:row0[t + 1]] = float("nan")
    o_d, x_d, g_d, tr0 = o_d.to(dev), x.to(dev), g.to(dev), S._i32(row0, dev)
    d_o, d_x = S._nan(N, d, dev=dev), S._nan(N, d, dev=dev)
    d_s = torch.full((T,), S.GARBAGE, device=dev)
    d_nw, d_nb = torch.full((T, d), S.GARBAGE, device=dev), torch.full((T, d), S.GARBAGE, device=dev)
    s_d = skip.to(dev) if skip is not None else None
    nw_d = nw.to(dev) if nw is not None else None
    perm_d = S._i32(perm, dev) if perm is not None else None
    act_d = S._i32(active, dev) if active is not None else None
    seed_d = _seed_tensor(seed, dev)
    common = (g_d.data_ptr(), o_d.data_ptr(), x_d.data_ptr(), tr0.data_ptr(), T, L.ptr(s_d), L.ptr(nw_d), L.ptr(perm_d),
              L.ptr(act_d), N, d, d_o.data_ptr(), d_x.data_ptr(), d_s.data_ptr(),
              d_nw.data_ptr() if nw is not None else None, d_nb.data_ptr() if nw is not None else None)
    guard_ok = True
    if det:
        need = ctypes.c_size_t()
        L.call("hgt_update_backward_det_workspace_bytes", N, T, d, ctypes.byref(need))
        buf = torch.full((need.value + 256,), 0xA5, dtype=torch.uint8, device=dev)
        L.call("hgt_update_backward_drop_det", *common, buf.data_ptr(), need.value, seed_d.data_ptr(), p, S._st())
        torch.cuda.synchronize()
        guard_ok = bool((buf[need.value:] == 0xA5).all())
    else:
        L.call("hgt_update_backward_drop", *common, seed_d.data_ptr(), p, S._st())
    torch.cuda.synchronize()
    return d_o.cpu(), d_x.cpu(), d_s.cpu(), d_nw.cpu(), d_nb.cpu(), guard_ok


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d", S.WIDTHS)
def test_update_backward_drop_matches_fp64(d, det):
    """Both backward kernels at every NPL, given the PRE-dropout o: d o = (float64 d (o * mask * s)) * mask * s, the
    rest as for the masked input; tolerances of test_update_backward_matches_fp64.  The deterministic and the atomic
    kernel draw the same mask: their d o agree in which elements are zero."""
    dev = _dev()
    p = 0.2
    o, x, g, skip, nw, perm_all = S._update_bwd_inputs(d, seed=3 * d + det)
    row0 = S._row0(S.BWD_COUNTS, S.BWD_UNKNOWN)
    N, T = row0[-1], len(S.BWD_COUNTS)
    mask = torch.from_numpy(drop_mask(SEED - d, N, d, p)).double() * float(drop_scale(p))
    o_eff = o.double() * mask
    for use_skip in (True, False):
        for use_norm in (True, False):
            for sharded in (False, True):
                s = skip if use_skip else None
                w = nw if use_norm else None
                perm = perm_all if sharded else None
                active = S.BWD_ACTIVE if sharded else None
                what = "d=%d det=%s skip=%s norm=%s perm/active=%s" % (d, det, use_skip, use_norm, sharded)
                d_o, d_x, d_s, d_nw, d_nb, guard_ok = _run_drop_bwd(o, x, g, s, w, perm, active, det, SEED - d, p, dev)
                ref = S._update_bwd_ref(o_eff.clone(), x, g, s, w, perm, active)      # it makes its input a leaf
                assert guard_ok, what
                for name, a, r in (("d_o", d_o, ref[0] * mask), ("d_x", d_x, ref[1])):
                    assert not torch.isnan(a).any(), what + ": %s has unwritten rows" % name
                    e = (S._scaled_max(a, r, 1.0), S._rel_fro(a, r, 1.0))
                    assert e[0] < 1.5e-4 and e[1] < 1e-4, (what, name, e)
                assert (d_o[mask == 0] == 0).all(), what + ": a dropped element has a gradient"
                if use_skip:
                    assert S._rel_fro(d_s, ref[2], 1.0) < 1.5e-4, (what, "d_skip")
                else:
                    assert (d_s == S.GARBAGE).all(), what
                if use_norm:
                    for name, a, r in (("d_norm_w", d_nw, ref[3]), ("d_norm_b", d_nb, ref[4])):
                        e = (S._scaled_max(a, r, 1.0), S._rel_fro(a, r, 1.0))
                        assert e[0] < 5e-6 and e[1] < 5e-6, (what, name, e)


# ---- layers -----------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _recorded_seeds():
    """Record the seed of every dropout site, in call order (the layers and the GNN draw them with autograd.drop_seed)."""
    from pyhgt_b200 import autograd, model
    seeds, real = [], autograd.drop_seed

    def rec(dev):
        s = real(dev)
        seeds.append(s)
        return s

    autograd.drop_seed = model.drop_seed = rec
    try:
        yield seeds
    finally:
        autograd.drop_seed = model.drop_seed = real


@contextlib.contextmanager
def _switch(on, *classes):
    old = [c.fused_dropout for c in classes]
    for c in classes:
        c.fused_dropout = on
    try:
        yield
    finally:
        for c, v in zip(classes, old):
            c.fused_dropout = v


class _Inject(torch.nn.Module):
    """Stands in for nn.Dropout: multiplies its k-th call's input by the k-th given multiplier (mask * s, fp32)."""
    def __init__(self, p, multipliers):
        super().__init__()
        self.p, self.multipliers = p, multipliers

    def forward(self, x):
        return x * self.multipliers.pop(0)


def test_hgtconv_matches_float64_with_the_mask_injected(monkeypatch):
    """out, d node_inp and every parameter gradient of one HGTConv training step with fused dropout against float64
    autograd through the oracle port, whose a_linear output is multiplied by the layer's own mask (conv.py:125)."""
    import pyhgt_b200
    from oracle import hgt_oracle
    dev = _dev()
    d, H, T, R, p = 128, 8, 3, 4, 0.2
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g = _graph(T, R, 5, True)
    torch.manual_seed(6)
    m = _perturb(pyhgt_b200.HGTConv(d, d, T, R, H, p, True, True), 7)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(8))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(9))
    params = _f64_params(m)
    m = m.to(dev).train()
    for det in (False, True):
        m.zero_grad()
        torch.use_deterministic_algorithms(det)
        try:
            with _switch(True, pyhgt_b200.HGTConv), _recorded_seeds() as seeds:
                native = _native_layer(m, x, g, w, dev)
        finally:
            torch.use_deterministic_algorithms(False)
        assert len(seeds) == 1
        mult = torch.from_numpy(drop_mask(int(seeds[0]), g.num_nodes, d, p)).double() * float(drop_scale(p))
        real = hgt_oracle._linear

        def linear(prm, name, t, inp):                  # sorted types: rank order is node order
            out = real(prm, name, t, inp)
            return out * mult[g.node_type == t] if name == "a_linears" else out

        for v in params.values():
            v.grad = None
        monkeypatch.setattr(hgt_oracle, "_linear", linear)
        xr = x.double().requires_grad_(True)
        out, _ = hgt_oracle.hgt_forward_ref_port(params, xr, g.node_type, g.edge_index, g.edge_type, g.edge_time,
                                                 num_types=T, num_relations=R, n_heads=H, use_norm=True, use_RTE=True)
        monkeypatch.setattr(hgt_oracle, "_linear", real)
        (out * w.double()).sum().backward()
        ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
        _compare_all("fused dropout det=%s" % det, native, ref, (1e-4, 1e-3))


def _gnn_case(kind, dev, p=0.2, n_layers=2, d=64):
    from pyhgt_b200.model import GNN
    T, R, f_in = 3, 4, 48
    g = _graph(T, R, 21, True, n_nodes=900, n_edges=6000)
    torch.manual_seed(3)
    gnn = _perturb(GNN(f_in, d, T, R, 4, n_layers, p, kind, True, True, True), 4).to(dev).train()
    x = torch.randn(g.num_nodes, f_in, generator=torch.Generator().manual_seed(5)).to(dev)
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(6)).to(dev)
    args = (g.node_type.to(dev), g.edge_time.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
    return gnn, x, w, args


def _gnn_step(gnn, x, w, args):
    gnn.zero_grad()
    xg = x.clone().requires_grad_(True)
    out = gnn(xg, *args)
    (out * w).sum().backward()
    torch.cuda.synchronize()
    return [out.detach().clone(), xg.grad.clone()] + [p.grad.clone() for p in gnn.parameters()]


def _classes():
    import pyhgt_b200
    from pyhgt_b200.model import GNN
    return pyhgt_b200.HGTConv, GNN


@pytest.mark.parametrize("kind", ["hgt", "dense_hgt"])
def test_gnn_matches_the_dropout_path_with_the_same_masks(kind, monkeypatch):
    """A 2-layer GNN (adapter + HGTConv or DenseHGTConv layers, two sites each for the latter) with the switch on
    against the same model with the switch off and every nn.Dropout replaced by a multiplication with the fused run's
    masks: the unfused path is the one the float64 gradient tests cover, so the two must agree to fp32 round-off."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    p = 0.2
    gnn, x, w, args = _gnn_case(kind, dev, p)
    with _switch(True, *_classes()), _recorded_seeds() as seeds:
        fused = _gnn_step(gnn, x, w, args)
    sites = 1 + (2 if kind == "dense_hgt" else 1) * len(gnn.gcs)
    assert len(seeds) == sites
    N, d = x.shape[0], gnn.n_hid
    mult = [(torch.from_numpy(drop_mask(int(s), N, d, p)).float() * float(drop_scale(p))).to(dev) for s in seeds]
    gnn.drop = _Inject(p, [mult[0]])
    k = 1
    for gc in gnn.gcs:
        n = 2 if kind == "dense_hgt" else 1
        gc.base_conv.drop = _Inject(p, mult[k:k + n])
        k += n
    plain = _gnn_step(gnn, x, w, args)
    names = ["out", "d x"] + [k_ for k_, _ in gnn.named_parameters()]
    for name, a, b in zip(names, fused, plain):
        # two fp32 evaluations of the same formulas, the atomic backward's summation order included
        assert S._rel_fro(a, b, 1e-6) < 5e-5, (kind, name, S._rel_fro(a, b, 1e-6))


def test_switch_is_inert_in_eval_and_at_p_zero(monkeypatch):
    """Switch on vs off gives bitwise equal outputs and gradients under eval() and at p = 0 (deterministic kernels, so
    two identical computations are bitwise equal); no seed is drawn in either."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    torch.use_deterministic_algorithms(True)
    try:
        for p, train in ((0.2, False), (0.0, True)):
            gnn, x, w, args = _gnn_case("hgt", dev, p)
            gnn.train(train)
            off = _gnn_step(gnn, x, w, args)
            with _switch(True, *_classes()), _recorded_seeds() as seeds:
                on = _gnn_step(gnn, x, w, args)
                with torch.no_grad():
                    on_ng = gnn(x, *args)
            with torch.no_grad():
                off_ng = gnn(x, *args)
            assert not seeds
            assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(on, off)), (p, train)
            assert torch.equal(_bits(on_ng), _bits(off_ng))
    finally:
        torch.use_deterministic_algorithms(False)


def test_same_torch_seed_same_gradients(monkeypatch):
    """torch.manual_seed reproduces the masks: two seeded steps under the deterministic flag are bitwise equal, another
    seed draws other masks.  The no_grad train-mode forward (conv.py per-stage path) draws the same masks as autograd's."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    gnn, x, w, args = _gnn_case("hgt", dev)
    torch.use_deterministic_algorithms(True)
    try:
        with _switch(True, *_classes()):
            torch.manual_seed(123)
            a = _gnn_step(gnn, x, w, args)
            torch.manual_seed(123)
            b = _gnn_step(gnn, x, w, args)
            torch.manual_seed(124)
            c = _gnn_step(gnn, x, w, args)
            torch.manual_seed(123)
            with torch.no_grad():
                ng = gnn(x, *args)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(_bits(u), _bits(v)) for u, v in zip(a, b))
    assert not torch.equal(a[0], c[0])
    # the inference kernels against the training forward: same masks, fp32 round-off apart
    assert S._rel_fro(ng, a[0]) < 2e-5


def test_training_step_holds_less_memory(monkeypatch):
    """Peak memory of one training step of a 2-layer GNN: with the switch on it is lower by at least the nn.Dropout
    masks of the layers (N * d bytes each)."""
    import pyhgt_b200
    from pyhgt_b200.model import GNN
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    T, R, d = 3, 4, 256
    g = _graph(T, R, 31, True, n_nodes=60000, n_edges=300000)
    torch.manual_seed(1)
    gnn = GNN(d, d, T, R, 8, 2, 0.2, "hgt", True, True, False).to(dev).train()
    x = torch.randn(g.num_nodes, d, device=dev)
    args = (g.node_type.to(dev), g.edge_time.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))
    peak = {}
    for on in (False, True, False, True):
        with _switch(on, *_classes()):
            for _ in range(2):                                        # the first step builds the plan and its tables
                gnn.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                gnn(x, *args).square().mean().backward()
                torch.cuda.synchronize()
                peak[on] = torch.cuda.max_memory_allocated() - base
    mask_bytes = len(gnn.gcs) * g.num_nodes * d
    print("\npeak memory of the step above its start: nn.Dropout %.1f MB, fused %.1f MB (layer masks %.1f MB)"
          % (peak[False] / 2 ** 20, peak[True] / 2 ** 20, mask_bytes / 2 ** 20))
    assert peak[True] <= peak[False] - mask_bytes, peak


# ---- captured training step -------------------------------------------------------------------------------------------
def test_graphed_step_draws_new_masks_and_freezes_the_switch(monkeypatch):
    import pyhgt_b200
    from pyhgt_b200 import graphed
    from tests import test_gpu_graphed_train as G
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    batches = G._batches()
    sig = G._signature(batches)
    gnn, head = G._model("hgt", dropout=0.5)
    rows = sig.type_counts[0]
    b = batches[0]
    y = G._labels(b)
    tens = (G._features(b), b.node_type, b.edge_time, b.edge_index, b.edge_type)
    with _switch(True, *_classes()):
        step = graphed.GraphedTrainStep(G._loss_fn(gnn, head, rows), sig, dev, targets={0: ((), torch.int64, -100)},
                                        params=list(gnn.parameters()) + list(head.parameters()))
        losses = [float(step(*tens, targets={0: y})[0]) for _ in range(4)]
        assert step.graph is not None
        assert len(set(losses[1:])) == 3, losses                      # replays 2-4: same batch, new masks
        gnn.gcs[0].base_conv.fused_dropout = False
        with pytest.raises(RuntimeError, match="fused_dropout"):
            step(*tens, targets={0: y})
        del gnn.gcs[0].base_conv.fused_dropout
        step(*tens, targets={0: y})
        gnn.fused_dropout = False
        with pytest.raises(RuntimeError, match="fused_dropout"):
            step(*tens, targets={0: y})


def test_graphed_sampled_minibatch_training_learns_with_fused_dropout():
    """The learnable sampled-minibatch task of tests/test_gpu_graphed_train.py (dropout 0.2, graphed, Adam), with the
    masks drawn in the kernels: same threshold."""
    import pyhgt_b200
    from pyhgt_b200 import data as hdata, graphed, sampler
    from pyhgt_b200.model import GNN
    from tests import test_gpu_graphed_train as G
    from tests.conftest import load_golden
    from tests.test_sampler import _GraphStub
    dev = _dev()
    fx = load_golden("sampler")
    g = _GraphStub(fx)
    fg = sampler.FrozenGraph(g)
    types = g.get_types()
    F_in, n_hid = 32, 64
    rng = np.random.RandomState(0)
    n_paper = fg.n_ids["paper"]
    venue_of = np.full(n_paper, -1, dtype=np.int64)
    for v, papers in fx["edge_list"]["venue"]["paper"]["PV_Journal"].items():
        for q in papers:
            venue_of[q] = v
    n_cls = int(venue_of.max()) + 1
    table = {t: rng.randn(fg.n_ids.get(t, 1), F_in).astype(np.float32) * 0.1 for t in types}
    table["paper"][np.arange(n_paper), np.clip(venue_of, 0, None) % F_in] += 1.0

    def extractor(layer_data, graph):
        feature, times, indxs = {}, {}, {}
        for _type in layer_data:
            if len(layer_data[_type]) == 0:
                continue
            idxs = np.array(list(layer_data[_type].keys()))
            feature[_type] = table[_type][idxs]
            times[_type] = np.array(list(layer_data[_type].values()))[:, 1]
            indxs[_type] = idxs
        return feature, times, indxs, []

    years = {}
    for a, papers in fx["edge_list"]["paper"]["author"]["AP_write"].items():
        for _author, t in papers.items():
            years[a] = t
    labelled = np.array([q for q in range(n_paper) if venue_of[q] >= 0 and q in years])
    edge_dict = {e[2]: i for i, e in enumerate(g.get_meta_graph())}
    edge_dict["self"] = len(edge_dict)
    Tn, Rn = len(types), len(edge_dict)
    data = []
    for step_i in range(40):
        np.random.seed(step_i)
        batch = np.random.choice(labelled, 32, replace=False)
        inp = {"paper": np.array([[int(q), int(years[q])] for q in batch])}
        feature, times, edge_list, _, _ = sampler.sample_subgraph(fg, fx["time_range"], 3, 12, inp, extractor)
        tens = hdata.to_torch(feature, times, edge_list, g, device=dev, prebuild_plan=True)
        data.append((tens[:5], torch.from_numpy(venue_of[batch]).to(dev)))
    sig, _ = G._device_signature(type("DG", (), {"types": types, "edge_dict": edge_dict, "feat_dim": F_in}),
                                 [d_[0] for d_ in data])
    paper = types.index("paper")
    old_att = pyhgt_b200.HGTConv.keep_att
    pyhgt_b200.HGTConv.keep_att = False
    try:
        with _switch(True, *_classes()):
            torch.manual_seed(0)
            gnn = GNN(F_in, n_hid, Tn, Rn, 4, 2, 0.2, "hgt", True, False, True).to(dev).train()
            head = torch.nn.Linear(n_hid, n_cls).to(dev)
            opt = torch.optim.Adam(list(gnn.parameters()) + list(head.parameters()), lr=2e-3, capturable=True)
            r0, C = int(sig.row0[paper]), sig.type_counts[paper]

            def loss_fn(x, nt, tm, ei, et, targets):
                return F.cross_entropy(head(gnn(x, nt, tm, ei, et)[r0:r0 + C]), targets[paper], ignore_index=-100)

            step = graphed.GraphedTrainStep(loss_fn, sig, dev, optimizer=opt, targets={paper: ((), torch.int64, -100)})
            losses = []
            for tens, y in data:
                loss, = step(*tens, targets={paper: y})
                losses.append(loss.clone())
            assert step.graph is not None and all(step.fused_drop.values()) and len(step.fused_drop) == 3
    finally:
        pyhgt_b200.HGTConv.keep_att = old_att
    losses = torch.stack(losses).cpu().numpy()
    assert np.isfinite(losses).all()
    assert np.mean(losses[-8:]) < 0.7 * np.mean(losses[:8]), losses
