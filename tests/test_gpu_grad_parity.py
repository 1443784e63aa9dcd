"""Training-path gradients against float64 autograd at the shapes the benchmarks run (run on an H100: ``pytest -m gpu``).

Each case builds an HGTConv in train() mode (dropout 0, att not kept) and runs the native training path on the GPU with
loss = sum(out * w) for a fixed seeded w.  The same parameters go through oracle.hgt_forward_ref_port in float64 under
torch autograd on the CPU; tests/test_oracle.py pins that float64 run to the reference's own gradient fixtures.  out,
d node_inp and the gradient of every named parameter are compared.  Every case runs twice: with linear_impl 0 (typed
GEMMs on the tensor cores wherever the shape allows) and with linear_impl 1 (fp32 SIMT GEMMs), so that a GEMM error can
be told apart from an edge-kernel or fold-kernel error.

The graphs have isolated destinations, self loops, duplicate edges and per-type node counts that are not multiples of
128, with one type of 37 nodes and one type with no nodes.  Two destinations lie above plan.TILE_SPLIT_EDGES, so the
split-destination path (k_merge_partials in the forward, atomic dq in the backward) runs at every head width.
"""
import contextlib
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hgt_oracle          # noqa: E402
from pyhgt_b200 import plan as P, synth  # noqa: E402

# name: (d, n_heads, num_types, num_relations, use_RTE, type-sorted node order).  The comments give the edge-backward
# instance k_edge_bwd<VEC, NCH> (csrc/edge_bwd.cu: LPH = 32 / next_pow2(H) lanes per head, VEC the widest of 4 / 2 / 1
# with d_k % VEC == 0 and d_k / VEC >= LPH, NCH = chunks per lane rounded up to a power of 2) and the output tile width
# BN of the tensor-core GEMMs (tc_ptx.cuh pick_tile_n; the dX / dW tiles of the backward use the same rule on K).
CASES = {
    "c2c4_d256_h8": (256, 8, 4, 4, False, True),      # d_k 32: <4,2>, red.global.add.v4.f32; BN 256, 4 k-blocks > 2 stages
    "c3_d400_h8_rte": (400, 8, 6, 10, True, False),   # d_k 50: <2,8>, chunk 6 partly and chunk 7 fully masked; BN 64 with
                                                      # a 16-column last tile, 7 k-blocks; RTE tables
    "c5_d128_h8": (128, 8, 4, 8, False, False),       # d_k 16: <4,1>; BN 128
    "dk25_d100_h4_rte": (100, 4, 3, 3, True, False),  # d_k 25: <1,4>; SIMT GEMMs in both runs (100 % 16 != 0)
    "h3_d96_rte": (96, 3, 3, 4, True, False),         # d_k 32: <4,1> with the lanes of a 4th head idle; BN 128, 2 k-blocks
    "h6_d384": (384, 6, 3, 3, False, False),          # d_k 64: <4,4>; BN 128 with 3 column tiles
    "h1_d256": (256, 1, 3, 2, False, False),          # d_k 256: LPH 32, <4,2>
    "h32_d256_rte": (256, 32, 3, 2, True, True),      # d_k 8: LPH 1, <4,2>
    "mag_d512_h8_rte": (512, 8, 4, 4, True, False),   # d_k 64: <4,4> with RTE on the fp32 register path (fewer than 2
                                                      # TMA ring stages fit); update NV 4 / NPL 16; BN 256, 2 column tiles
    "d1024_h8": (1024, 8, 3, 3, False, True),         # d_k 128: <4,8> (EDGE_UNROLL 1); update launch_vec<8>, NPL 32
    "h3_d78_rte": (78, 3, 3, 4, True, False),         # d_k 26: <2,2>; the scalar update epilogue (d % 4 != 0) and SIMT
                                                      # GEMMs in both runs (RTE's sinusoid table needs an even width)
}

# Relative-Frobenius bounds per tensor: (out and d node_inp, each parameter gradient), about 10x the worst error observed
# over both linear_impl runs on an H100 SXM (80 GB HBM3, 400 W power limit), which is given in the comment as
# (out / d node_inp, parameters).  impl 1 (fp32 SIMT) is 5-10x more accurate than impl 0; the bounds serve both.
# Parameter bounds above 1e-4: the worst tensor is relation_pri or skip.  Each of their entries is one sum of ~1e5 terms
# of mixed sign (d skip_t over the N_t x d outputs of type t; d relation_pri[r, h] over every <type, r> fold block of head
# h), so the ~1e-5 relative error of the split-bf16 GEMM outputs they are summed from comes back amplified by the
# cancellation.
FRO_BOUND = {
    "c2c4_d256_h8": (2e-5, 1e-4),        # 1.7e-6, 1.1e-5
    "c3_d400_h8_rte": (4e-5, 1e-4),      # 3.9e-6, 1.1e-5
    "c5_d128_h8": (2e-5, 2.5e-4),        # 1.6e-6, 2.3e-5 (skip)
    "dk25_d100_h4_rte": (2e-6, 2e-5),    # 1.6e-7, 1.5e-6 (both runs SIMT)
    "h3_d96_rte": (2e-5, 2e-4),          # 1.7e-6, 1.6e-5 (relation_pri)
    "h6_d384": (3e-5, 1e-4),             # 2.6e-6, 1.2e-5
    "h1_d256": (3e-5, 1.5e-4),           # 2.1e-6, 1.3e-5 (skip)
    "h32_d256_rte": (3e-5, 1.5e-4),      # 2.4e-6, 1.3e-5 (skip)
    "mag_d512_h8_rte": (4e-5, 1.5e-4),   # 3.7e-6, 1.2e-5
    "d1024_h8": (5e-5, 2e-4),            # 5.0e-6, 1.8e-5 (relation_pri)
    "h3_d78_rte": (2e-6, 2.5e-5),        # 1.4e-7, 2.3e-6 (skip; both runs SIMT)
}


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _type_counts(n_nodes, T):
    """Type 1 has no nodes, type 2 has 37; the rest share the remaining nodes.  None is a multiple of 128."""
    counts = [0] * T
    counts[2] = 37
    others = [t for t in range(T) if t not in (1, 2)]
    rest = n_nodes - 37
    for j, t in enumerate(others):
        counts[t] = rest // len(others) + 5 * j if j < len(others) - 1 else rest - sum(counts[o] for o in others[:-1])
    assert sum(counts) == n_nodes and all(c % 128 for c in counts if c)
    return counts


def _graph(T, R, seed, sorted_types, n_nodes=2400, n_edges=14000, hub_edges=(1500, 2600)):
    g = synth.make_random(n_nodes, n_edges, T, R, seed=seed, isolated_frac=0.1, self_loops=60, duplicate_edges=300)
    gen = torch.Generator().manual_seed(seed + 100)
    nt = torch.cat([torch.full((c,), t, dtype=torch.int64) for t, c in enumerate(_type_counts(n_nodes, T))])
    if not sorted_types:
        nt = nt[torch.randperm(n_nodes, generator=gen)]
    g.node_type = nt
    # destinations above the split threshold: 2 and 3 pieces at the default TILE_SPLIT_EDGES
    assert all(h > P.TILE_SPLIT_EDGES for h in hub_edges)
    hubs = [int((nt == 0).nonzero()[5]), int((nt == T - 1).nonzero()[3])]
    src, dst, rel, tm = [g.edge_index[0]], [g.edge_index[1]], [g.edge_type], [g.edge_time]
    for hub, cnt in zip(hubs, hub_edges):
        src.append(torch.randint(0, n_nodes, (cnt,), generator=gen))
        dst.append(torch.full((cnt,), hub, dtype=torch.int64))
        rel.append(torch.randint(0, R, (cnt,), generator=gen))
        tm.append(torch.randint(0, 240, (cnt,), generator=gen))
    g.edge_index = torch.stack([torch.cat(src), torch.cat(dst)])
    g.edge_type, g.edge_time = torch.cat(rel), torch.cat(tm)
    return g


def _perturb(m, seed):
    """Move the constant initialisations (skip, relation_pri, LayerNorm 1 / 0) away from their start values: a kernel that
    dropped one of these factors would otherwise compute the right numbers."""
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.rsplit(".", 1)[-1] in ("skip", "relation_pri") or ".norms." in "." + k:
                p.add_(0.3 * torch.randn(p.shape, generator=gen))
    return m


def _layer(d, H, T, R, rte, seed):
    import pyhgt_b200
    torch.manual_seed(seed)
    return _perturb(pyhgt_b200.HGTConv(d, d, T, R, H, 0.0, True, rte), seed + 1)


def _oracle_layer(params, x, g, m):
    out, _ = hgt_oracle.hgt_forward_ref_port(params, x, g.node_type, g.edge_index, g.edge_type,
                                             g.edge_time if m.use_RTE else None, num_types=m.num_types,
                                             num_relations=m.num_relations, n_heads=m.n_heads, use_norm=m.use_norm,
                                             use_RTE=m.use_RTE)
    return out


def _f64_params(m):
    return {k: p.detach().cpu().double().requires_grad_(True) for k, p in m.named_parameters()}


def _compare(got, ref, what, fro_bound):
    """allclose(rtol 1e-3, atol 1e-3 max|ref|) and relative Frobenius <= fro_bound against float64; returns the latter.
    A float64 gradient that is None or all zero (parameters of the type without nodes) needs an exact native zero."""
    if ref is None or not ref.abs().max().item():
        assert got is None or not got.abs().max().item(), \
            "%s: float64 gradient is zero, native max |g| %.3g" % (what, got.abs().max().item())
        return 0.0
    assert got is not None, "%s: no native gradient, float64 max |g| %.3g" % (what, ref.abs().max().item())
    got, ref = got.detach().cpu().double(), ref.detach().double()
    scale = ref.abs().max().item()
    fro = ((got - ref).norm() / ref.norm()).item()
    assert torch.isfinite(got).all(), "%s: non-finite values" % what
    assert torch.allclose(got, ref, rtol=1e-3, atol=1e-3 * scale), \
        "%s: max abs err %.3g (scale %.3g, rel fro %.3g)" % (what, (got - ref).abs().max().item(), scale, fro)
    assert fro <= fro_bound, "%s: relative Frobenius error %.3g > %.1g" % (what, fro, fro_bound)
    return fro


def _compare_all(tag, native, ref, bounds):
    """native / ref: (out, d node_inp, {parameter name: gradient}); bounds: (out and d node_inp, parameters).  Prints
    the worst errors (visible with -s)."""
    (o, dx, gp), (ro, rdx, rgp) = native, ref
    assert set(gp) == set(rgp)
    e_out = _compare(o, ro, tag + " out", bounds[0])
    e_dx = _compare(dx, rdx, tag + " d node_inp", bounds[0])
    worst, worst_k = 0.0, None
    for k in sorted(rgp):
        e = _compare(gp[k], rgp[k], "%s d %s" % (tag, k), bounds[1])
        if e >= worst:
            worst, worst_k = e, k
    print("\n%s: rel fro out %.2e, d node_inp %.2e, worst parameter %.2e (%s)" % (tag, e_out, e_dx, worst, worst_k))


_CACHE = {}


def _case(name):
    """Graph, layer state, input, loss weight and the float64 result of one case (computed once for both impls)."""
    if name not in _CACHE:
        d, H, T, R, rte, sorted_types = CASES[name]
        seed = sum(map(ord, name)) % 1000
        g = _graph(T, R, seed, sorted_types)
        m = _layer(d, H, T, R, rte, seed + 1)
        x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(seed + 2))
        w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(seed + 3))
        params = _f64_params(m)
        xr = x.double().requires_grad_(True)
        out = _oracle_layer(params, xr, g, m)
        (out * w.double()).sum().backward()
        ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
        _CACHE[name] = (g, m.state_dict(), x, w, ref)
    return _CACHE[name]


def _native_layer(m, x, g, w, dev):
    xg = x.to(dev).requires_grad_(True)
    out = m(xg, g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev) if m.use_RTE else None)
    (out * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    return out.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_layer_gradients_match_float64(name, impl, monkeypatch):
    """out, d node_inp and every parameter gradient of one HGTConv training step against float64 autograd.  The bounds
    and the worst errors observed on an H100 are listed per case at FRO_BOUND."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, state, x, w, ref = _case(name)
    d, H, T, R, rte, _ = CASES[name]
    m = pyhgt_b200.HGTConv(d, d, T, R, H, 0.0, True, rte)
    m.load_state_dict(state)
    m = m.to(dev).train()
    m.linear_impl = impl
    _compare_all("%s impl %d" % (name, impl), _native_layer(m, x, g, w, dev), ref, FRO_BOUND[name])


@pytest.mark.parametrize("impl", [0, 1])
def test_unmatched_edges_backward_matches_float64(impl, monkeypatch):
    """Training-path twin of test_out_of_range_relation_and_type_follow_reference_semantics: relation ids >= R and node
    types >= T mixed in, RTE on, d=256 / H=8.  Unmatched edges keep score 0 / message 0 in the destination's softmax;
    their dk / dv must land in the discarded trailing zero rows of the K'/V' and RTE gradient tables, not in a real row.
    A leak into an RTE row shows in the emb.lin gradients, a leak into a K'/V' row in the k / v / relation gradients.
    Nodes of unknown type get no gradient at all.  Worst relative Frobenius error observed on an H100: 2.2e-6 (out,
    d node_inp), 2.9e-5 (parameters: skip, see FRO_BOUND for why skip needs more than 1e-4)."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    T, R, d, H = 3, 4, 256, 8
    g = _graph(T, R, 61, False)
    g.edge_type[::7] = R + 5
    g.node_type[::11] = T + 2
    unknown = g.node_type >= T
    unmatched = unknown[g.edge_index[0]] | unknown[g.edge_index[1]] | (g.edge_type >= R)
    assert unmatched.sum() > 1000 and unknown.sum() > 100
    m = _layer(d, H, T, R, True, 62)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(63))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(64))
    params = _f64_params(m)
    xr = x.double().requires_grad_(True)
    out = _oracle_layer(params, xr, g, m)
    (out * w.double()).sum().backward()
    ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
    m = m.to(dev).train()
    m.linear_impl = impl
    native = _native_layer(m, x, g, w, dev)
    dx = native[1].cpu()
    assert (dx[unknown] == 0).all(), "nodes of unknown type got a gradient: max |dx| %.3g" % dx[unknown].abs().max()
    assert (native[0].cpu()[unknown] == 0).all()
    bounds = (3e-5, 3e-4)
    for k in ("emb.lin.weight", "emb.lin.bias"):
        _compare(native[2][k], ref[2][k], "unmatched edges impl %d d %s" % (impl, k), bounds[1])
    _compare_all("unmatched edges impl %d" % impl, native, ref, bounds)


# The GNN recipes: name -> (in_dim, n_hid, n_heads, n_layers, use_RTE), with prev_norm and last_norm on.  Their graphs
# are at _recipe_graph.  The bounds (out and d node_feature, parameters) are about 10x the worst relative Frobenius error
# observed over both linear_impl runs and both settings of the deterministic flag on an H100 SXM (80 GB HBM3, 400 W
# power limit), which the comment gives as (out / d node_feature, parameters).
RECIPES = {
    # 128 -> 256 into one HGTConv(256, 256, H=8) (edge backward <4,2>): the adapter's forward runs with BN 256, its dX
    # and dW with BN 128 over K = 128
    "adapter_128_256": ((128, 256, 8, 1, False), (5e-5, 1.5e-4)),      # 5.2e-6, 1.6e-5 (relation_pri)
    # ogbn-mag (reference ogbn-mag/train_ogbn_mag.py): K = 129, so the adapter's forward runs the padded-K tensor-core GEMM
    # (Kp = 136) and its backward the SIMT GEMMs (K % 16 != 0); edge <4,4> with RTE, on the fp32 register path
    # because fewer than 2 TMA ring stages fit
    "ogbn_mag": ((129, 512, 8, 4, True), (4e-5, 1.5e-4)),               # 3.8e-6, 1.5e-5 (relation_pri)
    # OAG (reference OAG/train_paper_venue.py and train_paper_field.py; train_author_disambiguation.py runs 3 layers):
    # in_dim 768 + 401 = 1169 (Kp = 1176), n_hid 400, edge <2,8>
    "oag": ((1169, 400, 8, 4, True), (8e-5, 2e-4)),                     # 8.1e-6, 1.8e-5 (skip)
    "oag_author_disambiguation": ((1169, 400, 8, 3, True), (8e-5, 2e-4)),  # 8.3e-6, 1.8e-5 (skip)
}


def _recipe_graph(name):
    if name == "ogbn_mag":
        # 1164 nodes of 4 types (institution 5), 12666 edges; Zipf destinations put two papers above TILE_SPLIT_EDGES
        return synth.make_mag_shaped(scale=6e-4, seed=2, dst_zipf=1.2)
    if name.startswith("oag"):
        return synth.make_oag_shaped(seed=3, n_nodes=1200, n_edges=7000)     # 6 types, 10 relations incl. 'self'
    return _graph(3, 4, 71, False)


def _oracle_gnn(params, x, g, m):
    """The GNN in float64: tanh(Linear_t(x)) (model.py:70-75), then hgt_forward_ref_port layer by layer."""
    h = torch.zeros(g.num_nodes, m.n_hid, dtype=torch.float64)
    for t in range(m.num_types):
        sel = g.node_type == t
        h[sel] = torch.tanh(x[sel] @ params["adapt_ws.%d.weight" % t].t() + params["adapt_ws.%d.bias" % t])
    for i, gc in enumerate(m.gcs):
        pre = "gcs.%d.base_conv." % i
        h = _oracle_layer({k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}, h, g, gc.base_conv)
    return h


def _recipe(name):
    """Graph, GNN state, input, loss weight and the float64 result of one recipe (computed once for every run)."""
    key = ("recipe", name)
    if key not in _CACHE:
        from pyhgt_b200.model import GNN
        (F_in, d, H, L, rte), _ = RECIPES[name]
        seed = sum(map(ord, name)) % 1000
        g = _recipe_graph(name)
        torch.manual_seed(seed)
        m = _perturb(GNN(F_in, d, g.num_types, g.num_relations, H, L, 0.0, "hgt", True, True, rte), seed + 1)
        x = torch.randn(g.num_nodes, F_in, generator=torch.Generator().manual_seed(seed + 2))
        w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(seed + 3))
        params = _f64_params(m)
        xr = x.double().requires_grad_(True)
        out = _oracle_gnn(params, xr, g, m)
        (out * w.double()).sum().backward()
        ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
        _CACHE[key] = (g, m, x, w, ref)
    return _CACHE[key]


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("recipe", list(RECIPES))
def test_gnn_adapter_projection_k_neq_width_matches_float64(recipe, impl, det, monkeypatch):
    """A GNN training step (typed input adapter tanh(Linear_t(x)) with K != width, then the HGTConv stack; dropout 0 in
    train mode) against float64 autograd: out, d node_feature and every parameter gradient, at the reference's own
    training recipes.  HGTConv itself needs in_dim == out_dim (the skip connection, conv.py:131), so the adapter is
    the training path's only projection with K != width.  Under torch.use_deterministic_algorithms two steps are
    bitwise equal."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, m0, x, w, ref = _recipe(recipe)
    m = copy.deepcopy(m0).to(dev).train()
    for c in m.gcs:
        c.base_conv.linear_impl = impl
    args = (g.node_type.to(dev), g.edge_time.to(dev), g.edge_index.to(dev), g.edge_type.to(dev))

    def step():
        m.zero_grad(set_to_none=True)
        xg = x.to(dev).requires_grad_(True)
        o = m(xg, *args)
        (o * w.to(dev)).sum().backward()
        torch.cuda.synchronize()
        return o.detach(), xg.grad, {k: p.grad for k, p in m.named_parameters()}

    with _deterministic(det):
        native = step()
        again = step() if det else None
    _compare_all("GNN %s impl %d det %d" % (recipe, impl, det), native, ref, RECIPES[recipe][1])
    if det:
        assert torch.equal(native[0], again[0]) and torch.equal(native[1], again[1])
        for k, v in native[2].items():
            assert (v is None and again[2][k] is None) or torch.equal(v, again[2][k]), k


def test_c4_three_layer_stack_matches_float64(monkeypatch):
    """The workload bench.py c4 times: three HGTConv(256, 256, 4, 4, 8, 0.0, True, False) layers chained, forward and
    backward on the tensor-core path, against the float64 oracle applied layer by layer (graph of the c2c4 case).
    Worst relative Frobenius error observed on an H100: 4.4e-6 (out, d node_inp), 1.2e-5 (parameters)."""
    import pyhgt_b200
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    g, _, x, w, _ = _case("c2c4_d256_h8")
    layers = torch.nn.ModuleList([_layer(256, 8, 4, 4, False, 80 + 2 * i) for i in range(3)])
    params = [_f64_params(m) for m in layers]
    xr = x.double().requires_grad_(True)
    h = xr
    for p, m in zip(params, layers):
        h = _oracle_layer(p, h, g, m)
    (h * w.double()).sum().backward()
    ref = (h.detach(), xr.grad, {"%d.%s" % (i, k): v.grad for i, p in enumerate(params) for k, v in p.items()})
    layers = layers.to(dev).train()
    xg = x.to(dev).requires_grad_(True)
    nt, ei, et = g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev)
    h = xg
    for m in layers:
        h = m(h, nt, ei, et)
    (h * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    native = (h.detach(), xg.grad, {k: p.grad for k, p in layers.named_parameters()})
    _compare_all("c4 stack", native, ref, (5e-5, 1e-4))
