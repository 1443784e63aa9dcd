"""Training gradients on the whole ogbn-mag-shaped c2 graph (N = 1.94 M, E = 21.1 M, d = 256) against float64 (run on
an H100: ``pytest -m gpu``).

At this size the flat projection buffer [Q | K'/V'] holds 1.12 x 2^31 fp32 elements and the bf16 K'/V' table of
autocast passes 2^31 bytes, so every product that indexes them (the edge backward's row offsets, the bf16 hi/lo split of
the projection gradient, the dX / dW jobs, the in-place row pass of recompute_tables) must be 64-bit.  The smaller
training tests never reach these offsets.

Technique (the gradient form of test_gpu_parity._sampled_rows_vs_oracle): the loss is sum(out[S] * w_S) for a seeded
destination set S (tests/test_full_graph_train_cpu.py:full_graph_sample).  An L-layer stack's loss depends only on the
L-hop in-neighbourhood R_L of S, so oracle.hgt_forward_ref_port in float64 on the subgraph induced by R_L gives the
exact out[S], d node_inp on R_L and every parameter gradient.  Every backward stage maps a zero upstream gradient to
exact zeros, so the native d node_inp must be exactly zero outside R_L: a stray write or a misaddressed read anywhere in
the 2.4e9-element buffers shows there.  Misaddressing produces O(1) errors, which the float64 comparison catches in every
precision mode.

`-s` prints the worst relative Frobenius error and the peak memory (max_memory_allocated) of every case.  Observed on an
H100 80GB HBM3 at 700 W, as (out / d node_inp, parameters): one layer 5.9e-7, 1.2e-5 (peaks: keep 30.3 / 30.8 GB, lean
32.4 / 32.5 GB with the deterministic flag off / on); the c4 stack 1.4e-6, 3.5e-5 (51.2 / 51.3 GB); the hubs 1.7e-6,
4.4e-5 (36.1 GB).
"""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

import pyhgt_b200                                                                       # noqa: E402
from oracle import hgt_oracle                                                           # noqa: E402
from pyhgt_b200 import plan as P, synth                                                 # noqa: E402
from tests.test_full_graph_train_cpu import (D, full_graph_sample, hub_destinations, kv_rows_of,  # noqa: E402
                                             projection_layout, HUB_PIECE_EDGES)
from tests.test_fused_dropout_cpu import drop_mask_rows, drop_scale                      # noqa: E402
from tests.test_gpu_bf16_tables import OUT_MAX_ABS as BF16_OUT_MAX_ABS, OUT_REL_FRO as BF16_OUT_REL_FRO  # noqa: E402
from tests.test_gpu_fused_dropout import _recorded_seeds, _switch                        # noqa: E402
from tests.test_gpu_grad_parity import FRO_BOUND, _compare_all, _f64_params, _layer, _oracle_layer, _perturb  # noqa: E402
from tests.test_gpu_matmul_precision import (GRAD_REL_FRO as MEDIUM_GRAD_REL_FRO,       # noqa: E402
                                             OUT_MAX_ABS as MEDIUM_OUT_MAX_ABS, OUT_REL_FRO as MEDIUM_OUT_REL_FRO,
                                             _precision, _rel)
from tests.test_gpu_recompute_tables import _det                                        # noqa: E402

H, T, R = 8, 4, 4
BOUND = FRO_BOUND["c2c4_d256_h8"]
BF16_GRAD_REL_FRO = 5e-2           # test_gpu_bf16_tables.test_conv_training_step_under_bf16_autocast
DROP_BOUND = (1e-4, 1e-3)          # test_gpu_fused_dropout.test_hgtconv_matches_float64_with_the_mask_injected
STACK_BOUND = (5e-5, 1e-4)         # test_gpu_grad_parity.test_c4_three_layer_stack_matches_float64


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


class _Graph:
    """One full-size graph on the GPU with its input, and the float64 results computed for it so far."""

    def __init__(self, g, dev):
        self.g, self.dev = g, dev
        self.nt, self.ei, self.et, self.tm = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev),
                                              g.edge_time.to(dev))
        self.x = torch.randn(g.num_nodes, D, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        self.cache = {}

    def args(self, rte):
        return (self.nt, self.ei, self.et, self.tm if rte else None)

    def close(self):
        self.__dict__.clear()
        P.clear_plan_cache()
        gc.collect()
        torch.cuda.empty_cache()


def _module_graph(g):
    c = _Graph(g, _dev())
    try:
        yield c
    finally:
        c.close()


@pytest.fixture(scope="module")
def c2():
    yield from _module_graph(synth.make_mag_shaped(1.0, seed=2))


@pytest.fixture(scope="module")
def zipf():
    yield from _module_graph(synth.make_mag_shaped(1.0, seed=2, dst_zipf=1.1))


def _weights(s, seed):
    return torch.randn(s.S.numel(), D, generator=torch.Generator().manual_seed(seed))


def _sample(c, layers):
    key = ("sample", layers)
    if key not in c.cache:
        c.cache[key] = full_graph_sample(c.g, layers)
    return c.cache[key]


def _native(c, model, forward, s, w, tag, det=False, autocast=False, precision="highest"):
    """One training step of `model` on the whole graph with loss sum(out[S] * w): (out[S], d node_inp on R_L, {parameter:
    gradient}) on the host.  Asserts that d node_inp is exactly zero outside R_L and prints the step's peak memory."""
    dev = c.dev
    model.zero_grad(set_to_none=True)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    S, nodes = s.S.to(dev), s.nodes.to(dev)
    xg = c.x.detach().requires_grad_(True)
    with _det(det), _precision(precision):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = forward(xg)
        assert out.dtype == torch.float32
        out_s = out[S]
        del out
        (out_s * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 1e9
    dx = xg.grad
    dx_rows = dx[nodes].cpu()
    dx[nodes] = 0
    stray = (dx != 0).any(1).nonzero(as_tuple=True)[0]
    assert stray.numel() == 0, "%s: d node_inp is nonzero at %d rows outside R_L, e.g. %s (max |g| %.3g)" % (
        tag, stray.numel(), stray[:8].tolist(), dx.abs().max().item())
    grads = {k: None if p.grad is None else p.grad.detach().cpu() for k, p in model.named_parameters()}
    del dx, xg
    print("\n%s: peak memory %.1f GB" % (tag, peak))
    return out_s.detach().cpu(), dx_rows, grads


def _reference(c, mods, s, w, prefix=lambda i: ""):
    """float64 autograd through the oracle port, layer by layer, on the subgraph of `s`."""
    params = [_f64_params(m) for m in mods]
    xr = c.x[s.nodes.to(c.dev)].cpu().double().requires_grad_(True)
    h = xr
    for p, m in zip(params, mods):
        h = _oracle_layer(p, h, s.sub, m)
    rows = s.local[s.S]
    (h[rows] * w.double()).sum().backward()
    return (h[rows].detach(), xr.grad, {prefix(i) + k: v.grad for i, p in enumerate(params) for k, v in p.items()})


def _layer_on(c, m, lean):
    m = m.to(c.dev).train()
    m.keep_att = False
    m.recompute_tables = lean
    return m


def _one_layer(c, m, lean):
    m = _layer_on(c, m, lean)
    return m, lambda xg: m(xg, *c.args(m.use_RTE))


def _plain(c, mode, det):
    """The fp32 HGTConv(256, 256, 4, 4, 8, 0.0, True, False) step in keep or lean mode (cached per graph) and the
    float64 result it is held to."""
    key = ("plain", mode, det)
    if key not in c.cache:
        s, w = _sample(c, 1), _weights(_sample(c, 1), 3)
        layer = _layer(D, H, T, R, False, 11)
        if "plain_ref" not in c.cache:
            c.cache["plain_ref"] = _reference(c, [layer], s, w)
        m, fwd = _one_layer(c, layer, mode == "lean")
        tag = "c2 1 layer %s det %d" % (mode, det)
        c.cache[key] = _native(c, m, fwd, s, w, tag, det=det)
        _compare_all(tag, c.cache[key], c.cache["plain_ref"], BOUND)
    return c.cache[key]


def _assert_bitwise(a, b, tag):
    assert torch.equal(a[0], b[0]), "%s: out[S]" % tag
    assert torch.equal(a[1], b[1]), "%s: d node_inp" % tag
    assert set(a[2]) == set(b[2])
    bad = [k for k in sorted(a[2]) if not ((a[2][k] is None and b[2][k] is None) or torch.equal(a[2][k], b[2][k]))]
    assert not bad, "%s: gradients differ: %s" % (tag, bad)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the layout the offsets come from

def test_projection_layout_matches_the_library(c2):
    """The host restatement (pairs, pair_row0, kv_rows, kv_off, proj_elems, and every sampled edge's K'/V' row) is the
    layout the library builds, so the offsets the CPU file asserts are the ones the kernels use."""
    plan = P.get_plan(c2.nt, c2.ei, c2.et, None, T, R)
    lay = projection_layout(c2.g, D)
    assert plan.pairs == lay["pairs"] and plan.pair_row0 == lay["pair_row0"] and plan.kv_rows == lay["kv_rows"]
    lt = P.layer_tables(plan, D, D)
    assert (lt.kv_off, lt.proj_elems) == (lay["kv_off"], lay["proj_elems"]) and lt.proj_elems > 2 ** 31
    s = _sample(c2, 1)
    kv_by_edge = torch.empty(plan.n_edges, dtype=torch.int32, device=c2.dev)
    kv_by_edge[plan.csr_eid[:plan.n_edges].long()] = plan.kv_row[:plan.n_edges]
    assert torch.equal(kv_by_edge[s.edges.to(c2.dev)].long().cpu(), kv_rows_of(c2.g, lay, s.edges))
    del kv_by_edge


# ---------------------------------------------------------------------------------------------------------------------
# 2. one layer on the whole c2 graph

@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("mode", ["keep", "lean"])
def test_one_layer_matches_float64(c2, mode, det):
    """fp32, dropout 0, no RTE, in keep mode and in lean mode (recompute_tables), with the deterministic flag off and
    on: out[S], d node_inp on R_1 and every parameter gradient against float64, exact zeros elsewhere."""
    _plain(c2, mode, det)


def test_keep_and_lean_are_bitwise_equal_under_the_deterministic_flag(c2):
    """DESIGN.md §5 claims this at c4; here at the full c2 size (d node_inp outside R_1 is zero in both)."""
    _assert_bitwise(_plain(c2, "keep", True), _plain(c2, "lean", True), "keep vs lean at full size")


def test_one_layer_with_rte_matches_float64(c2):
    """Lean, deterministic flag on, RTE on (the generator's edge_time): the RTE-row pass and its table gradients."""
    s = _sample(c2, 1)
    w = _weights(s, 4)
    layer = _layer(D, H, T, R, True, 12)
    ref = _reference(c2, [layer], s, w)
    m, fwd = _one_layer(c2, layer, True)
    tag = "c2 1 layer rte lean det 1"
    _compare_all(tag, _native(c2, m, fwd, s, w, tag, det=True), ref, BOUND)


def test_one_layer_with_fused_dropout_matches_float64(c2, monkeypatch):
    """Lean, deterministic flag on, fused_dropout at p = 0.2: the oracle's a_linear output is multiplied by the layer's
    own mask (tests/test_fused_dropout_cpu.py), drawn for the subgraph's rows only.  The c2 node ids are type-sorted, so
    a node's rank row is its id."""
    s = _sample(c2, 1)
    w = _weights(s, 5)
    p = 0.2
    torch.manual_seed(13)
    layer = _perturb(pyhgt_b200.HGTConv(D, D, T, R, H, p, True, False), 14)
    params = _f64_params(layer)
    m, fwd = _one_layer(c2, layer, True)
    tag = "c2 1 layer fused dropout lean det 1"
    with _switch(True, pyhgt_b200.HGTConv), _recorded_seeds() as seeds:
        native = _native(c2, m, fwd, s, w, tag, det=True)
    assert len(seeds) == 1
    mult = torch.from_numpy(drop_mask_rows(int(seeds[0]), s.nodes.numpy(), D, p)).double() * float(drop_scale(p))
    assert 0.7 < float((mult > 0).double().mean()) < 0.9
    real = hgt_oracle._linear

    def linear(prm, name, t, inp):
        out = real(prm, name, t, inp)
        return out * mult[s.sub.node_type == t] if name == "a_linears" else out

    monkeypatch.setattr(hgt_oracle, "_linear", linear)
    xr = c2.x[s.nodes.to(c2.dev)].cpu().double().requires_grad_(True)
    out = _oracle_layer(params, xr, s.sub, layer)
    monkeypatch.setattr(hgt_oracle, "_linear", real)
    rows = s.local[s.S]
    (out[rows] * w.double()).sum().backward()
    _compare_all(tag, native, (out[rows].detach(), xr.grad, {k: v.grad for k, v in params.items()}), DROP_BOUND)


@pytest.mark.parametrize("kind", ["bf16_autocast", "medium"])
def test_one_layer_low_precision_stays_close_to_fp32(c2, kind):
    """Lean under bf16 autocast (bf16 K'/V' table past byte 2^31) and at float32 matmul precision "medium", against
    the fp32 full-graph run of the same layer with the bounds of test_gpu_bf16_tables / test_gpu_matmul_precision;
    the exact-zero rule holds too."""
    s = _sample(c2, 1)
    ref = _plain(c2, "lean", False)
    m, fwd = _one_layer(c2, _layer(D, H, T, R, False, 11), True)
    tag = "c2 1 layer lean %s" % kind
    if kind == "bf16_autocast":
        got = _native(c2, m, fwd, s, _weights(s, 3), tag, autocast=True)
        out_max, out_fro, grad_fro = BF16_OUT_MAX_ABS, BF16_OUT_REL_FRO, BF16_GRAD_REL_FRO
    else:
        got = _native(c2, m, fwd, s, _weights(s, 3), tag, precision="medium")
        out_max, out_fro, grad_fro = MEDIUM_OUT_MAX_ABS, MEDIUM_OUT_REL_FRO, MEDIUM_GRAD_REL_FRO
    assert not torch.equal(got[0], ref[0]), "%s: the low-precision path did not run" % tag
    err = float((got[0] - ref[0]).abs().max())
    fro = {"out": _rel(got[0], ref[0]), "d node_inp": _rel(got[1], ref[1])}
    assert err <= out_max and fro["out"] <= out_fro, "%s: out max-abs %.3g, rel fro %.3g" % (tag, err, fro["out"])
    for k, g in ref[2].items():
        if g is None or not g.abs().max().item():
            assert got[2][k] is None or not got[2][k].abs().max().item(), "%s: d %s should be zero" % (tag, k)
            continue
        fro["d " + k] = _rel(got[2][k], g)
    worst = max(fro, key=fro.get)
    print("\n%s: vs fp32 out max-abs %.2e; worst rel fro %.2e (%s)" % (tag, err, fro[worst], worst))
    bad = {k: v for k, v in fro.items() if k != "out" and v > grad_fro}
    assert not bad, "%s: gradients past rel fro %.0e: %s" % (tag, grad_fro, bad)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the advertised step: the c4 stack on the whole c2 graph

@pytest.mark.parametrize("det", [False, True])
def test_c4_stack_lean_on_the_whole_graph_matches_float64(c2, det):
    """3 x HGTConv(256, 256, 4, 4, 8, 0.0, True, False) in lean mode, the step README and DESIGN.md §5 report for the
    whole graph: out[S], d node_inp on R_3 (exact zeros elsewhere) and every layer's parameter gradients against
    float64 on the 3-hop field.  With the deterministic flag on a second step is bitwise equal.  DESIGN.md §5 measured
    a 54.5 GB peak with the flag off; -s prints this run's."""
    s = _sample(c2, 3)
    w = _weights(s, 6)
    layers = torch.nn.ModuleList([_layer(D, H, T, R, False, 80 + 2 * i) for i in range(3)])
    if "stack_ref" not in c2.cache:
        c2.cache["stack_ref"] = _reference(c2, list(layers), s, w, prefix=lambda i: "%d." % i)
    for m in layers:
        _layer_on(c2, m, True)

    def fwd(xg):
        h = xg
        for m in layers:
            h = m(h, *c2.args(False))
        return h

    tag = "c2 c4 stack lean det %d" % det
    native = _native(c2, layers, fwd, s, w, tag, det=det)
    _compare_all(tag, native, c2.cache["stack_ref"], STACK_BOUND)
    if det:
        _assert_bitwise(native, _native(c2, layers, fwd, s, w, tag + " (second step)", det=True), tag)


# ---------------------------------------------------------------------------------------------------------------------
# 4. hub destinations at full size

@pytest.mark.parametrize("det", [False, True])
def test_hub_destinations_at_full_size_match_float64(zipf, det):
    """make_mag_shaped(1.0, dst_zipf=1.1), lean, one layer: S holds the heaviest destination below 10^5 in-edges (about
    95 hub pieces), another with 10^4 .. 10^5, and ordinary ones, so thousands of hub pieces of the whole graph run
    through the atomic-dq / piece-merge paths while the sampled ones are checked.  The heaviest destination (1.13 M
    in-edges) stays out on purpose: each per-edge float64 tensor of its subgraph is 2.3 GB, so its float64 run would
    need 20 GB or more of host memory."""
    if "hub_sample" not in zipf.cache:
        (h1, h2), deg = hub_destinations(zipf.g)
        s = full_graph_sample(zipf.g, 1, counts=(4, 2, 4, 1), extra=(h1, h2), max_in_edges=HUB_PIECE_EDGES)
        assert int(deg[s.S].max()) // HUB_PIECE_EDGES >= 10 and int((deg > HUB_PIECE_EDGES).sum()) > 1000
        zipf.cache["hub_sample"] = s
    s = zipf.cache["hub_sample"]
    w = _weights(s, 7)
    layer = _layer(D, H, T, R, False, 21)
    if "hub_ref" not in zipf.cache:
        zipf.cache["hub_ref"] = _reference(zipf, [layer], s, w)
    m, fwd = _one_layer(zipf, layer, True)
    tag = "c2 zipf 1.1 hubs lean det %d" % det
    _compare_all(tag, _native(zipf, m, fwd, s, w, tag, det=det), zipf.cache["hub_ref"], BOUND)
