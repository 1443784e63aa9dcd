"""bs16 [K'|V'] and RTE gather tables (include/hgt_b200.h, "bs16 gather tables") on the GPU.

- The typed GEMM's bs16 output (hgt_typed_linear[_presplit]_bs16) is the fp32 call's output encoded by the numpy
  restatement (tests/test_bs16_format_cpu.py), bitwise, at every forward instance: 64 / 128 / 256-column tiles, three
  products and one, fp32 and presplit A, the mixed Q + table job, padded column blocks, and the SIMT kernel.
- hgt_edge_forward_bs16 equals hgt_edge_forward on the decoded table bitwise (it decodes each element to m * s, an exact
  fp32 value, and keeps the fp32 kernel's arithmetic), at every lane map, with and without RTE, on both data paths,
  and on sync-free plans with poisoned tails.
- The format rule: small (L2-resident) tables stay 24-bit, the full-size c2 table is bs16, and hgt_conv_forward and
  the per-stage path pick the same format and agree bitwise.
"""
import ctypes

import numpy as np
import pytest
import torch

from pyhgt_b200 import _lib
from tests.test_bs16_format_cpu import decode, encode, row_bytes
from tests.test_gpu_bf16_tables import _conv, _dev, _gemm_table, _inputs, _st
from tests.test_gpu_edge_instances import SHAPES, _plan, _q_scale, _tables, lane_map, ring_fallback
from tests.test_gpu_t24_tables import T24_EXTRA_SHAPES, _edge, _record

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# 1. typed GEMM with a bs16 output

@pytest.mark.parametrize("mixed", [False, True])
@pytest.mark.parametrize("path,K,width,ms,shared", [
    ("tc2", 64, 64, [200, 37, 128], False),           # BN = 64 (staged epilogue)
    ("tc2", 96, 128, [300, 129], False),              # BN = 128 (tensor stores)
    ("tc2", 128, 256, [150, 257], False),             # BN = 256
    ("tc2", 64, 80, [150, 70], False),                # BN = 128, columns 80..127 of each block padded
    ("tc2", 64, 240, [150, 70], False),               # BN = 256, scales of the V' block not 8-byte aligned: staged
    ("tc2", 64, 400, [333, 64], False),               # d = 400: BN = 64, last tile masked
    ("tc2", 64, 64, [17 + 5 * i for i in range(70)], False),   # more than 64 groups: chunked launches
    ("tc3", 64, 64, [200, 37], False),                # one bf16 product
    ("tc3", 128, 256, [150, 257], False),
    ("presplit", 64, 64, [200, 37, 128], False),
    ("presplit", 96, 128, [300, 129], False),
    ("presplit", 128, 256, [150, 257], False),
    ("presplit", 64, 400, [333, 64], False),
    ("presplit1", 128, 256, [150, 257], False),       # a_lo = NULL: one product
    ("simt", 64, 64, [240, 240, 240], True),          # RTE tables: overlapping groups on the SIMT kernel
    ("simt", 48, 208, [240, 240], True),
])
def test_gemm_bs16_output_equals_encoded_fp32(path, K, width, ms, shared, mixed):
    """mixed: the first group's column blocks lie before the table offset and are written as fp32 (the Q blocks of a
    projection), the others into the bs16 table; otherwise every block is bs16."""
    dev = _dev()
    tab, rows, out_elems, w_rows = _gemm_table(K, width, ms, shared)
    off = ms[0] * 2 * width if mixed else 0
    n = 2 * width
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator().manual_seed(K + width + len(ms))
    a = (torch.randn(rows, K, generator=gen) * 3).to(dev)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    # a few whole rows of W zero (zero blocks), one scaled far up and one far down
    w[1] = 0
    w[2] *= 1e30
    w[3] *= 1e-30
    out32 = torch.zeros(out_elems, device=dev)
    n_rows = (out_elems - off) // n
    out16 = torch.full((n_rows * row_bytes(n),), 0xAB, dtype=torch.uint8, device=dev)
    out_q = torch.zeros(off, device=dev) if mixed else None
    outs = {"fp32": (out32.data_ptr(),), "bs16": (_lib.ptr(out_q), off, out16.data_ptr())}
    wsb = ctypes.c_size_t()
    if path.startswith("presplit"):
        hi = a.to(torch.bfloat16)
        lo = None if path == "presplit1" else (a - hi.float()).to(torch.bfloat16)
        _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, kind in (("hgt_typed_linear_presplit", "fp32"), ("hgt_typed_linear_presplit_bs16", "bs16")):
            _lib.call(fn, hi.data_ptr(), _lib.ptr(lo), w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(),
                      g_host.ctypes.data, n_g, c_dev.data_ptr(), *outs[kind], ws.data_ptr(), ws.numel(), _st())
    else:
        impl = {"tc2": 2, "tc3": 3, "simt": 1}[path]
        _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        for fn, kind in (("hgt_typed_linear", "fp32"), ("hgt_typed_linear_bs16", "bs16")):
            _lib.call(fn, a.data_ptr(), K, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(), g_host.ctypes.data,
                      n_g, c_dev.data_ptr(), *outs[kind], impl, ws.data_ptr(), ws.numel(), _st())
    torch.cuda.synchronize()
    assert out32.abs().max() > 0
    got = out16.view(n_rows, row_bytes(n)).cpu().numpy()[:, :2 * n + n // 8]
    want = encode(out32[off:].view(n_rows, n).cpu().numpy())[:, :2 * n + n // 8]
    assert np.array_equal(got, want)
    if mixed:
        assert torch.equal(out_q, out32[:off])


# ---------------------------------------------------------------------------------------------------------------------
# 2. the edge forward on bs16 tables

BS16_SHAPES = sorted({(d, H) for d, H in SHAPES + T24_EXTRA_SHAPES if d % 16 == 0} |
                     {(144, 2), (144, 8), (96, 2), (48, 16), (112, 16), (240, 16)})


def test_bs16_shapes_reach_every_lane_map():
    every = {(v, n) for v in (1, 2, 4) for n in (1, 2, 4, 8)}
    assert {lane_map(d, H) for d, H in BS16_SHAPES} == every, every - {lane_map(d, H) for d, H in BS16_SHAPES}


def _encode_dev(x):
    return torch.from_numpy(encode(x.cpu().numpy()).reshape(-1)).to(x.device)


def _decode_dev(t, n):
    return torch.from_numpy(decode(t.cpu().numpy(), n)).to(t.device)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("rte", [False, True])
@pytest.mark.parametrize("d,H", BS16_SHAPES)
def test_edge_forward_bs16_equals_fp32_on_decoded(d, H, rte, variant):
    plan, T = _plan(d, H, rte, seed=d + H)
    q, kv, kvr = _tables(plan, d, rte, d, torch.float32, _q_scale(d, H, False))
    kv16 = _encode_dev(kv)
    kvr16 = None if kvr is None else _encode_dev(kvr)
    kv_dec = _decode_dev(kv16, 2 * d)
    kvr_dec = None if kvr is None else _decode_dev(kvr16, 2 * d)
    # bitwise where both calls take the same data path: the ring where the fp32 rows fit it (the bs16 rows, smaller,
    # then fit too), the register gather where both keep as many rows in flight (bs16 keeps half the fp32 kernel's)
    vec, nch = lane_map(d, H)
    unroll = [(1 if w >= 32 else 2 if w >= 16 else 4) for w in (2 * vec * nch, vec * nch)]
    same_path = ring_fallback(d, H, rte, 4) is None if variant == 2 else unroll[0] == unroll[1]
    has_in = (plan.row_ptr[1:] - plan.row_ptr[:-1]) > 0
    for gelu in (False, True):
        got = _edge("hgt_edge_forward_bs16", plan, T, q, kv16, kvr16, d, H, variant, gelu)
        want = _edge("hgt_edge_forward", plan, T, q, kv_dec, kvr_dec, d, H, variant, gelu)
        torch.cuda.synchronize()
        for name, a, b in zip(("agg", "att", "stats", "g_hi", "g_lo"), got, want):
            if a is None:
                continue
            if name == "stats":
                a, b = a[has_in], b[has_in]
            if same_path:
                assert torch.equal(a, b), (name, gelu)
            elif name in ("agg", "att", "stats"):            # another order of the same sums (the bf16 split of
                torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)   # gelu(agg) follows agg, a rounding apart)


@pytest.mark.parametrize("variant", [1, 2])
def test_edge_forward_bs16_sync_free_poisoned_tails(variant):
    """Sync-free plans: the grid is sized for an upper bound of tiles, the device count says how many are real, and
    the tile entries past it are poison.  The bs16 kernel reads only the real ones, as the fp32 kernel does."""
    d, H = 256, 8
    plan, T = _plan(d, H, False, seed=5)
    q, kv, _ = _tables(plan, d, False, d, torch.float32, _q_scale(d, H, False))
    kv16 = _encode_dev(kv)
    kv_dec = _decode_dev(kv16, 2 * d)
    n_real = plan.n_tiles
    tiles = torch.full((n_real + 64, 4), -7, dtype=torch.int32, device=q.device)
    tiles[:n_real] = plan.tiles.view(-1, 4)[:n_real]
    counts = torch.tensor([n_real, plan.n_split, plan.n_hubs], dtype=torch.int32, device=q.device)
    saved = plan.tiles, plan.n_tiles, plan.tile_counts_dev
    try:
        plan.tiles, plan.n_tiles, plan.tile_counts_dev = tiles.view(-1), n_real + 64, counts
        got = _edge("hgt_edge_forward_bs16", plan, T, q, kv16, None, d, H, variant, False)
        want = _edge("hgt_edge_forward", plan, T, q, kv_dec, None, d, H, variant, False)
    finally:
        plan.tiles, plan.n_tiles, plan.tile_counts_dev = saved
    torch.cuda.synchronize()
    if variant == 2:                                         # the same ring: bitwise
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    else:                                                    # the register gather keeps fewer bs16 rows in flight
        torch.testing.assert_close(got[0], want[0], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(got[1], want[1], rtol=1e-4, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the rule

def test_rule_thresholds():
    l2 = torch.cuda.get_device_properties(_dev()).L2_cache_size
    rows = l2 // (6 * 256)
    assert _lib.gather_table_format(256, rows, _dev()) == _lib.TABLE_T24
    assert _lib.gather_table_format(256, rows + 1, _dev()) == _lib.TABLE_BS16
    assert _lib.gather_table_format(264, 10 ** 7, _dev()) == _lib.TABLE_T24       # d % 128 != 0
    assert _lib.gather_table_format(400, 10 ** 7, _dev()) == _lib.TABLE_T24       # c3: staged epilogue, stays 24-bit
    assert _lib.gather_table_format(128, 10 ** 7, _dev()) == _lib.TABLE_BS16
    assert _lib.gather_table_format(100, 10 ** 7, _dev()) == _lib.TABLE_F32


def test_c1_fixture_stays_t24(conv_fixture, monkeypatch):
    fx, dev = conv_fixture, _dev()
    m = _conv(fx, dev)
    args = _inputs(fx, dev)
    names = _record(monkeypatch)
    with torch.no_grad():
        m(*args)
    assert not any(n.endswith("_bs16") for n in names)


def test_large_table_fused_and_staged_pick_bs16_and_agree(monkeypatch):
    """A graph whose 24-bit table is larger than L2: both inference paths build bs16 tables and agree bitwise."""
    import pyhgt_b200
    from pyhgt_b200 import synth
    dev = _dev()
    g = synth.make_mag_shaped(0.1)
    d = 256
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, g.num_types, g.num_relations, 8, 0.0, True, False).to(dev).eval()
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1)).to(dev)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), None)
    names = _record(monkeypatch)
    with torch.no_grad():
        fused = m(x, *args)
    assert "hgt_conv_forward" in names
    names.clear()
    pyhgt_b200.HGTConv.event_sink = []
    try:
        with torch.no_grad():
            staged = m(x, *args)
    finally:
        pyhgt_b200.HGTConv.event_sink = None
    assert "hgt_edge_forward_bs16" in names and "hgt_typed_linear_bs16" in names
    assert torch.equal(fused, staged)
