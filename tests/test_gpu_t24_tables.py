"""24-bit [K'|V'] and RTE gather tables (include/hgt_b200.h, "24-bit gather tables") on the GPU.

- The typed GEMM's 24-bit output (hgt_typed_linear[_presplit]_t24) is the fp32 call's output encoded, bitwise, at every
  instance: 64 / 128 / 256-column tiles, three products and one, fp32 and presplit A, group tails, padded column blocks,
  the SIMT kernel, and the projection table of the full-size ogbn-mag-shaped graph.
- hgt_edge_forward_t24 equals hgt_edge_forward on the decoded table bitwise (the decoded words are fp32 values, and the
  lane map and arithmetic are the same), for both data paths, with RTE, hub splits, att and the gelu hi/lo output; and
  float64 on the decoded table at the fp32 instances' tolerance.
- A no-grad HGTConv forward (24-bit tables) stays within MAX_ABS / REL_FRO of a grad-recording forward (fp32 tables)
  of the same module, on the C1 fixtures and on sampled rows of the full-size c2, c3 and c5 graphs; the fused call and
  the per-stage path agree bitwise.
"""
import ctypes

import numpy as np
import pytest
import torch

from pyhgt_b200 import _lib, plan as P, synth
from tests.test_gpu_bf16_tables import _conv, _dev, _gemm_table, _inputs, _rel, _st
from tests.test_gpu_edge_instances import (HOT_SHAPES, SHAPES, _check_hot, _edge_ref, _plan, _q_scale, _tables, lane_map,
                                           ring_fallback)
from tests.test_t24_format_cpu import encode

pytestmark = pytest.mark.gpu

# Deviation of a layer's output with 24-bit tables from the fp32-table forward: about 17x / 12x the float64 estimate
# of rounding only K'/V' (5.8e-6 max-abs, 8.1e-7 relative Frobenius on the 1 % ogbn-mag-shaped graph)
MAX_ABS, REL_FRO = 1e-4, 1e-5


def round_words(x):
    """torch restatement of tests/test_t24_format_cpu.round_bits on any device: float32 -> rounded words (int64)."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    special = (b & 0x7F800000) == 0x7F800000
    nan = special & ((b & 0x7FFFFF) != 0)
    r = torch.where(special, b, (b + 0x7F + ((b >> 8) & 1)) & 0xFFFFFF00)
    return torch.where(nan, (b | 0x400000) & 0xFFFFFF00, r)


def words(t, n):
    """uint8 [rows * 3n] planar 24-bit rows -> the stored words as int64 [rows, n]."""
    t = t.view(-1, 3 * n)
    hi = t[:, :2 * n].contiguous().view(torch.int16).to(torch.int64) & 0xFFFF
    return (hi << 16) | (t[:, 2 * n:].to(torch.int64) << 8)


def decode(t, n):
    """uint8 planar rows -> float32 [rows, n]."""
    w = words(t, n)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32).view(torch.float32)


def encode_t(x):
    """float32 [rows, n] -> uint8 [rows * 3n] planar rows, on x's device."""
    r = round_words(x)
    hi = (r >> 16).to(torch.int32).to(torch.int16)           # low 16 bits, little-endian bytes
    lo = ((r >> 8) & 0xFF).to(torch.uint8)
    return torch.cat([hi.view(torch.uint8).view(x.shape[0], -1), lo], 1).reshape(-1)


def test_torch_restatement_matches_numpy():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(33, 40, generator=gen) * torch.exp(torch.randn(33, 40, generator=gen) * 10)
    x.view(-1)[:4] = torch.tensor([float("inf"), -float("inf"), float("nan"), 0.0])
    x.view(-1)[4:6] = torch.tensor([0x7F800001, 0x007FFFFF], dtype=torch.int32).view(torch.float32)
    assert np.array_equal(encode_t(x.to(_dev())).cpu().numpy(), encode(x.numpy()).reshape(-1))


# ---------------------------------------------------------------------------------------------------------------------
# 1. typed GEMM with a 24-bit output

@pytest.mark.parametrize("mixed", [False, True])
@pytest.mark.parametrize("path,K,width,ms,shared", [
    ("tc2", 64, 64, [200, 37, 128], False),           # BN = 64
    ("tc2", 96, 128, [300, 129], False),              # BN = 128
    ("tc2", 128, 256, [150, 257], False),             # BN = 256
    ("tc2", 64, 80, [150, 70], False),                # BN = 128, columns 80..127 of each block padded
    ("tc2", 64, 400, [333, 64], False),               # d = 400: BN = 64, last tile masked
    ("tc2", 64, 64, [17 + 5 * i for i in range(70)], False),   # more than 64 groups: chunked launches
    ("tc3", 64, 64, [200, 37], False),                # one bf16 product
    ("tc3", 128, 256, [150, 257], False),
    ("tc3", 96, 128, [300, 129], False),
    ("presplit", 64, 64, [200, 37, 128], False),
    ("presplit", 96, 128, [300, 129], False),
    ("presplit", 128, 256, [150, 257], False),
    ("presplit", 64, 400, [333, 64], False),
    ("presplit1", 128, 256, [150, 257], False),       # a_lo = NULL: one product
    ("presplit1", 64, 64, [200, 37], False),
    ("simt", 64, 64, [240, 240, 240], True),          # RTE tables: overlapping groups on the SIMT kernel
    ("simt", 48, 200, [240, 240], True),
])
def test_gemm_t24_output_equals_encoded_fp32(path, K, width, ms, shared, mixed):
    """mixed: the first group's column blocks lie before t24_off and are written as fp32 (the Q blocks of a projection
    table), the others as 24-bit; otherwise every block is 24-bit."""
    dev = _dev()
    tab, rows, out_elems, w_rows = _gemm_table(K, width, ms, shared)
    t24_off = ms[0] * 2 * width if mixed else 0
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator().manual_seed(K + width + len(ms))
    a = (torch.randn(rows, K, generator=gen) * 3).to(dev)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    out32 = torch.zeros(out_elems, device=dev)
    out24 = torch.zeros(3 * (out_elems - t24_off), dtype=torch.uint8, device=dev)
    out_q = torch.zeros(t24_off, device=dev) if mixed else None
    outs = {"fp32": (out32.data_ptr(),), "t24": (_lib.ptr(out_q), t24_off, out24.data_ptr())}
    wsb = ctypes.c_size_t()
    if path.startswith("presplit"):
        hi = a.to(torch.bfloat16)
        lo = None if path == "presplit1" else (a - hi.float()).to(torch.bfloat16)
        _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, kind in (("hgt_typed_linear_presplit", "fp32"), ("hgt_typed_linear_presplit_t24", "t24")):
            _lib.call(fn, hi.data_ptr(), _lib.ptr(lo), w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(),
                      g_host.ctypes.data, n_g, c_dev.data_ptr(), *outs[kind], ws.data_ptr(), ws.numel(), _st())
    else:
        impl = {"tc2": 2, "tc3": 3, "simt": 1}[path]
        _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, kind in (("hgt_typed_linear", "fp32"), ("hgt_typed_linear_t24", "t24")):
            _lib.call(fn, a.data_ptr(), K, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data,
                      n_g, c_dev.data_ptr(), *outs[kind], impl, ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    assert out32.abs().max() > 0
    assert torch.equal(words(out24, 2 * width), round_words(out32[t24_off:].view(-1, 2 * width)))
    if mixed:
        assert torch.equal(out_q, out32[:t24_off])


def test_c2_projection_table_equals_encoded_fp32():
    """The projection of the full-size ogbn-mag-shaped graph (d = 256): Q as fp32 and the K'/V' blocks (7.7 GB as fp32,
    5.7 GB as 24-bit, byte offsets past 2^32) from one call, against the fp32 call, compared in row chunks."""
    dev, d = _dev(), 256
    g = synth.make_mag_shaped(1.0)
    plan = P.build_plan(g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), None, g.num_types,
                        g.num_relations)
    lt = P.layer_tables(plan, d, d)
    g_dev, g_host, n_g, c_dev = lt.proj_groups
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(plan.n_nodes, d, generator=gen).to(dev)
    w = (torch.randn(lt.cat_rows, d, generator=gen) / 16).to(dev)
    b = torch.randn(lt.cat_rows, generator=gen).to(dev)
    n_rows = plan.kv_rows
    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, d, d, 2, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    q24 = torch.empty(lt.kv_off, device=dev)
    out24 = torch.empty(n_rows * 6 * d, dtype=torch.uint8, device=dev)
    _lib.call("hgt_typed_linear_t24", x.data_ptr(), d, w.data_ptr(), b.data_ptr(), d, d, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), q24.data_ptr(), lt.kv_off, out24.data_ptr(), 2, ws.data_ptr(),
              ws.numel(), _st())
    proj = torch.empty(lt.kv_off + n_rows * 2 * d, device=dev)
    _lib.call("hgt_typed_linear", x.data_ptr(), d, w.data_ptr(), b.data_ptr(), d, d, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), proj.data_ptr(), 2, ws.data_ptr(), ws.numel(), _st())
    assert n_rows * 6 * d > 2 ** 32
    assert torch.equal(q24[:plan.n_nodes * d], proj[:plan.n_nodes * d])
    t24, t32 = out24.view(n_rows, 6 * d), proj[lt.kv_off:].view(n_rows, 2 * d)
    for r0 in range(0, n_rows, 1 << 20):
        assert torch.equal(words(t24[r0:r0 + (1 << 20)], 2 * d), round_words(t32[r0:r0 + (1 << 20)])), r0


# ---------------------------------------------------------------------------------------------------------------------
# 2. the edge forward on 24-bit tables

T24_SHAPES = [(d, H) for d, H in SHAPES if d % 8 == 0]
# d % 8 == 0 shapes for the two lane maps the shared lists reach only with d % 8 != 0: <1,4> (d_k 9) and <2,2> (d_k 36)
T24_EXTRA_SHAPES = [(72, 8), (72, 2)]
T24_HOT_SHAPES = [(d, H) for d, H in HOT_SHAPES if d % 8 == 0] + T24_EXTRA_SHAPES


def _edge(fn, plan, T, q, kv, kvr, d, H, variant, gelu):
    """agg (or gelu(agg)), att, stats and the bf16 hi/lo split of one edge forward."""
    dev = q.device
    N, E = plan.n_nodes, plan.n_edges
    agg = torch.full((N, d), float("nan"), device=dev)
    att = torch.empty(E, H, device=dev)
    stats = torch.empty(N, 2 * H, device=dev)
    g_hi = torch.empty(N, d, dtype=torch.bfloat16, device=dev) if gelu else None
    g_lo = torch.empty(N, d, dtype=torch.bfloat16, device=dev) if gelu else None
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    _lib.call(fn, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
              plan.rte_row.data_ptr() if kvr is not None else None, plan.csr_eid.data_ptr(), plan.tiles.data_ptr(),
              plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, N, E, d, H, int(gelu), agg.data_ptr(),
              att.data_ptr(), stats.data_ptr(), _lib.ptr(g_hi), _lib.ptr(g_lo), ws.data_ptr(), ws.numel(), variant,
              _lib.ptr(plan.tile_counts_dev), plan.type_row0_dev.data_ptr(), T, None, _st())
    return agg, att, stats, g_hi, g_lo


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("rte", [False, True])
@pytest.mark.parametrize("d,H", T24_SHAPES)
def test_edge_forward_t24(d, H, rte, variant):
    _check_edge_forward_t24(d, H, rte, variant, False)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("rte", [False, True])
@pytest.mark.parametrize("d,H", T24_EXTRA_SHAPES)
def test_edge_forward_t24_extra_lane_maps(d, H, rte, variant):
    _check_edge_forward_t24(d, H, rte, variant, False)


def test_t24_shape_lists_reach_every_lane_map():
    """The 24-bit forward runs (and its (m, l) is checked against float64) at all 12 <VEC, NCH> lane maps, with
    ordinary and with hot scores."""
    every = {(v, n) for v in (1, 2, 4) for n in (1, 2, 4, 8)}
    assert {lane_map(d, H) for d, H in T24_SHAPES + T24_EXTRA_SHAPES} == every
    assert {lane_map(d, H) for d, H in T24_HOT_SHAPES} == every
    assert all(d % 8 == 0 for d, _ in T24_HOT_SHAPES + T24_EXTRA_SHAPES)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("d,H", T24_HOT_SHAPES)
def test_edge_forward_t24_hot(d, H, variant):
    """Hot scores (most exp terms underflow in fp32): the online rescale and the hub pieces' merge on 24-bit rows."""
    _check_edge_forward_t24(d, H, True, variant, True)


def _check_edge_forward_t24(d, H, rte, variant, hot):
    plan, T = _plan(d, H, rte, seed=d + H)
    assert plan.n_split > 0
    q, kv, kvr = _tables(plan, d, rte, d, torch.float32, _q_scale(d, H, hot))
    kv24 = encode_t(kv)
    kvr24 = None if kvr is None else encode_t(kvr)
    kv_dec = decode(kv24, 2 * d)
    kvr_dec = None if kvr is None else decode(kvr24, 2 * d)
    # the same kernel as the fp32 call on the decoded table: then the same arithmetic in the same order, bitwise.  Not
    # so where a 6d-byte row leaves room for a ring that an 8d-byte row does not, nor where the register gather keeps
    # fewer 24-bit rows in flight (csrc/edge.cu, EDGE_UNROLL)
    vec, nch = lane_map(d, H)
    ldg = variant == 1 or ring_fallback(d, H, rte, 3) is not None
    unroll = [(1 if w >= 32 else 2 if w >= 16 else 4) for w in (2 * vec * nch, vec * nch)]
    same_path = (ring_fallback(d, H, rte, 3) == ring_fallback(d, H, rte, 4) or variant == 1) and \
        not (ldg and unroll[0] != unroll[1])
    for gelu in (False, True):
        got = _edge("hgt_edge_forward_t24", plan, T, q, kv24, kvr24, d, H, variant, gelu)
        if not same_path:
            continue
        want = _edge("hgt_edge_forward", plan, T, q, kv_dec, kvr_dec, d, H, variant, gelu)
        torch.cuda.synchronize()
        has_in = (plan.row_ptr[1:] - plan.row_ptr[:-1]) > 0
        for name, a, b in zip(("agg", "att", "stats", "g_hi", "g_lo"), got, want):
            if a is not None:
                if name == "stats":
                    a, b = a[has_in], b[has_in]
                assert torch.equal(a, b), (name, gelu)
    ref, att_ref, m_ref, l_ref = _edge_ref(plan, q.cpu().double(), kv_dec.cpu().double(),
                                           None if kvr_dec is None else kvr_dec.cpu().double(), H)
    if hot:
        _check_hot(att_ref)
    agg, att, stats = got[0], got[1], got[2].cpu().double()
    # the tolerances of tests/test_gpu_edge_instances.py (hot: the rounding error of a score grows with its size)
    atol = 1e-4 if hot else 1e-5
    torch.testing.assert_close(agg.cpu().double(), torch.nn.functional.gelu(ref), rtol=1e-4, atol=atol)
    eid = plan.csr_eid[:plan.n_edges].cpu().long()
    torch.testing.assert_close(att.cpu().double()[eid], att_ref, rtol=1e-4, atol=1e-6)
    has_in = ((plan.row_ptr[1:] - plan.row_ptr[:-1]) > 0).cpu()
    torch.testing.assert_close(stats[:, :H][has_in], m_ref[has_in], rtol=1e-5, atol=atol)
    torch.testing.assert_close(stats[:, H:][has_in], l_ref[has_in], rtol=1e-4, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# 3. layers

def _record(monkeypatch):
    names = []
    real = _lib.call

    def call(name, *args):
        names.append(name)
        return real(name, *args)
    monkeypatch.setattr(_lib, "call", call)
    return names


def _within_bounds(got, ref, what):
    err, fro = float((got - ref).abs().max()), _rel(got, ref)
    assert torch.isfinite(got).all() and err <= MAX_ABS and fro <= REL_FRO, \
        "%s: max-abs %.3g, rel-Frobenius %.3g" % (what, err, fro)
    return err, fro


def test_conv_fixture_no_grad_against_fp32_tables(conv_fixture, monkeypatch):
    """No-grad (24-bit tables where d % 8 == 0, fp32 tables otherwise; fused call and per-stage path bitwise equal)
    against a grad-recording forward (fp32 tables)."""
    import pyhgt_b200
    fx, dev = conv_fixture, _dev()
    m = _conv(fx, dev)
    t24 = m.out_dim % 8 == 0
    args = _inputs(fx, dev)
    names = _record(monkeypatch)
    with torch.no_grad():
        fused = m(*args)
    assert "hgt_conv_forward" in names
    names.clear()
    pyhgt_b200.HGTConv.event_sink = []
    try:
        with torch.no_grad():
            staged = m(*args)
    finally:
        pyhgt_b200.HGTConv.event_sink = None
    assert ("hgt_edge_forward_t24" in names) == t24 and ("hgt_edge_forward" in names) != t24
    assert torch.equal(fused, staged)
    names.clear()
    x = args[0].clone().requires_grad_(True)
    ref = m(x, *args[1:]).detach()
    assert "hgt_edge_forward_t24" not in names and not any(n.endswith("_t24") for n in names)
    _within_bounds(fused, ref, fx["name"])


@pytest.mark.parametrize("config", ["c2", "c3", "c5"])
def test_full_size_no_grad_against_fp32_tables(config):
    """One layer on the benchmark's full-size graphs: the 24-bit forward against the fp32-table forward of the same
    module, on 200 k sampled rows (all rows are computed; the comparison is sampled to bound host memory)."""
    import pyhgt_b200
    dev = _dev()
    d, rte, g = {"c2": (256, False, lambda: synth.make_mag_shaped(1.0)),
                 "c3": (400, True, lambda: synth.make_oag_shaped(1.0)),
                 "c5": (128, False, lambda: synth.make_powerlaw(64_000_000))}[config]
    g = g()
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, g.num_types, g.num_relations, 8, 0.0, True, rte).to(dev).eval()
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1)).to(dev)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev) if rte else None)
    rows = torch.randperm(g.num_nodes, generator=torch.Generator().manual_seed(2))[:200_000].to(dev)
    with torch.no_grad():
        got = m(x, *args)[rows]
    ref = m(x.clone().requires_grad_(True), *args).detach()[rows]
    err, fro = _within_bounds(got, ref, config)
    print("%s: max-abs %.3g rel-Frobenius %.3g" % (config, err, fro))
