"""Every compiled instance of the typed-GEMM backward (csrc/linear_bwd.cu) against float64 on the same tables.

hgt_typed_linear_bwd / hgt_typed_linear_bwd_det run either on the tensor cores (k_lin_dx_tc, k_lin_dw_tc and, in
deterministic mode, k_lin_dw_tc_det, each compiled at 64-, 128- and 256-column tiles and with three or one bf16
products; the dOut split pass k_split_colsum / k_split_colsum_det in front of them) or on the fp32 SIMT kernels
(k_lin_dx_simt, k_lin_dw_simt and their deterministic twins).  `bwd_instance` restates that choice (bwd_layout,
bwd_tc_ok, pick_tile_n and typed_linear_bwd), and test_case_list_reaches_every_instance (no GPU needed) checks that CASES
reaches every kernel, every reason for the SIMT path and deterministic dW reductions of three or more row chunks.

Each case is checked against float64 autograd of sum(dout * (act(A) W^T + b)) over its column-block table, built here
from the header's formulas.  Three products and SIMT are held to an elementwise bound on the scale of each output
(|dout| @ |W| for dA, |dout|^T @ |A| for dW, sum |dout| for db); one product is compared with float64 of the
bf16-rounded operands at the tolerance of test_gpu_matmul_precision.py.  The calls start from sentinels: dW and db are
prefilled with random values (they are accumulated into), dA with NaN (rows between groups must come back 0, rows past the
last group stay NaN) or, with accumulate_dA, with random values.  Every case also runs with each of dA, dW and db NULL,
and the deterministic entry point runs every case twice, bitwise equal.
"""
import ctypes
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

from pyhgt_b200 import _lib

BF16 = torch.bfloat16
BM, BK = 128, 64                   # tensor-core tile rows / k-block (tc_ptx.cuh)
DW_SIMT_ROWS = 2048                # rows per SIMT dW chunk (linear_bwd.cu)
H100_SMS = 132                     # SMs of an H100 SXM: the deterministic tensor-core dW chunks depend on it
# Elementwise error bounds, as a fraction of the scale of each output element.  One product: the products of the
# bf16-rounded operands are exact in fp32, only the fp32 accumulation remains (test_gpu_matmul_precision.ACC_TOL).
# Three products drop lo*lo and what the lo halves do not hold: bf16 keeps 8 significant bits, so up to about
# 3 * 2^-16 of |a w| for a single term (a dW row of a one-row group).  On an H100 the worst ratio seen was 2.1e-5 (P = 3),
# 3.8e-7 (P = 1) and 3.7e-7 (SIMT).
TOL = {1: 1e-5, 3: 5e-5, None: 1e-5}          # keyed by the number of bf16 products; None: fp32 SIMT


# ---------------------------------------------------------------------------------------------------------------------
# the kernel-selection rule, restated

def pick_tile_n(k):
    """tc_ptx.cuh pick_tile_n: the widest of 64 / 128 / 256 columns that pads k no more than a narrower one."""
    best, best_pad = 64, -(-k // 64) * 64
    for bn in (128, 256):
        pad = -(-k // bn) * bn
        if pad <= best_pad:
            best, best_pad = bn, pad
    return best


def _overlap(groups):
    live = [(a0, a0 + m) for a0, m, *_ in groups if m > 0]
    return any(a < d and c < b for i, (a, b) in enumerate(live) for c, d in live[i + 1:])


def simt_reason(K, width, groups, cblocks, lda):
    """Why bwd_tc_ok sends a table to the SIMT kernels (its checks in order), or None."""
    if width % 8:
        return "width % 8"
    if K % 16:
        return "K % 16"
    if K < 64:
        return "K < 64"
    if width < 16:
        return "width < 16"
    if lda != K:
        return "lda != K"
    if _overlap(groups):
        return "overlap"
    for _, _, _, ncb, cb0, _ in groups:
        if any(off % 8 or ld % 8 for off, ld in cblocks[cb0:cb0 + ncb]):
            return "align"
    if sum(g[1] for g in groups) < 512:
        return "rows < 512"
    return None


def tc_dw_chunk(task_rows, width, K, sms):
    tn = pick_tile_n(K)
    chunk = task_rows * -(-width // BM) * -(-K // tn) // (4 * sms)
    return min(max(-(-chunk // BK) * BK, 1024), 32768)


def simt_det_chunk(task_rows):
    chunk = -(-task_rows // 256)
    return max(-(-chunk // 32) * 32, DW_SIMT_ROWS)


# tile_n: the width of the dX and of the dW tiles (both pick_tile_n(K)); P: bf16 products (None on SIMT)
Instance = namedtuple("Instance", "tc reason tile_n P split dw_chunks kernels")


def bwd_instance(K, width, groups, cblocks, lda, impl, dsplit, asplit, det, sms=H100_SMS):
    """The path, tiles, products, split pass, deterministic dW chunks per task and kernel instances of one call with
    dA, dW and db all given.  groups: (a_row0, m, w_row0, n_cblocks, cb_first, has_bias); cblocks: (out_off, ld)."""
    reason = "impl 1" if impl == 1 else simt_reason(K, width, groups, cblocks, lda)
    tc = impl == 2 or (impl == 3 and asplit) or (impl in (0, 3) and reason is None)
    if tc:
        reason = None
    P = (1 if impl == 3 else 3) if tc else None
    tn = pick_tile_n(K)
    split = None
    if tc and not dsplit:
        split = "k_split_colsum_det" if det else "k_split_colsum"
    chunks = None
    if det:
        task_rows = sum(g[1] * g[3] for g in groups)
        chunk = tc_dw_chunk(task_rows, width, K, sms) if tc else simt_det_chunk(task_rows)
        chunks = max(-(-g[1] // chunk) for g in groups)
    sfx = "_det" if det else ""
    if tc:
        kernels = {("k_lin_dx_tc", tn, P), ("k_lin_dw_tc" + sfx, tn, P)}
    else:
        kernels = {("k_lin_dx_simt" + sfx,), ("k_lin_dw_simt" + sfx,)}
    if split:
        kernels.add((split,))
    return Instance(tc, reason, tn, P, split, chunks, kernels)


# ---------------------------------------------------------------------------------------------------------------------
# cases

Case = namedtuple("Case", "K width spec layout impl lda_pad misalign gelu asplit dsplit share_w")


def C(K, width, spec, layout="pairs", impl=0, lda_pad=0, misalign=False, gelu=False, asplit=False, dsplit=False,
      share_w=False):
    """spec: [(rows, column blocks, has_bias)].  layout "pairs": a group's first column block in a [rows, width] region,
    the others interleaved two by two in [rows, 2 * width] regions (ld = 2 * width: the projection's K'/V' layout);
    "single": every column block in its own [rows, width] region; "rte": every group projects rows 0..rows of the same A
    (overlapping groups, like the RTE tables)."""
    return Case(K, width, spec, layout, impl, lda_pad, misalign, gelu, asplit, dsplit, share_w)


CASES = {
    # the benchmark layers; c2c4 has a group of 3,001 rows (three deterministic dW chunks) and groups of 129, 0 and 1
    "c2c4": C(256, 256, [(3001, 3, 1), (129, 1, 0), (0, 1, 1), (1, 2, 1)]),
    "c2c4_p1": C(256, 256, [(65, 3, 1), (3100, 1, 1), (127, 2, 0)], impl=3),
    # c3: 64-wide dX / dW tiles, 7 column tiles, and 400 - 3 * 128 = 16 rows in the last dW m-tile
    "c3": C(400, 400, [(900, 3, 1), (65, 1, 0), (64, 2, 1)]),
    "c3_p1": C(400, 400, [(600, 3, 1), (63, 1, 1)], impl=3, gelu=True),
    "c5": C(128, 128, [(63, 1, 1), (64, 2, 0), (127, 1, 1), (300, 3, 1)], layout="single"),
    "c5_p1": C(128, 128, [(129, 3, 1), (400, 1, 1)], impl=3, layout="single"),
    # K = 80: 128-wide dX tiles, the last k-block of W^T / A is 16 columns wide
    "k80": C(80, 64, [(600, 2, 1), (129, 1, 1)]),
    # widths only the backward takes on the tensor cores
    "w16": C(256, 16, [(300, 3, 1), (250, 1, 0)]),
    "w24_p1": C(192, 24, [(400, 2, 1), (200, 1, 1)], impl=3),
    "w40": C(128, 40, [(520, 3, 1)], gelu=True),
    # split_colsum over 260 float4 columns (more than its 256 threads)
    "w1040": C(64, 1040, [(520, 1, 1), (1, 1, 1)], layout="single"),
    "gelu_c2": C(256, 256, [(2049, 1, 1), (513, 1, 1)], layout="single", gelu=True),
    # groups that share W rows (the sharded per-pair compaction): dW / db of both land in the same rows
    "shared_w": C(128, 128, [(700, 2, 1), (300, 2, 1)], share_w=True),
    # operands split by their producers: A hi + lo (impl 2), A hi only (impl 3), dOut hi + lo / hi only (no db)
    "asplit": C(256, 256, [(1000, 3, 1), (130, 1, 1)], impl=2, asplit=True, gelu=True),
    "asplit_p1": C(128, 128, [(800, 3, 1)], impl=3, asplit=True),
    "dsplit": C(256, 256, [(1000, 3, 1), (130, 1, 1)], dsplit=True),
    "dsplit_p1": C(400, 400, [(700, 1, 1)], impl=3, dsplit=True, asplit=True),
    # SIMT, one case per reason
    "simt_w20": C(64, 20, [(4500, 2, 1), (30, 1, 0)]),                 # also three deterministic dW chunks
    "simt_k1169": C(1169, 32, [(200, 1, 1), (150, 2, 1)], gelu=True),
    "simt_k48": C(48, 32, [(700, 2, 1)]),
    "simt_w8": C(64, 8, [(700, 3, 1)]),
    "simt_lda": C(64, 64, [(700, 2, 1)], lda_pad=8),
    "simt_rte": C(64, 64, [(240, 2, 0)] * 5 + [(240, 2, 1)], layout="rte", gelu=True),
    "simt_align": C(64, 64, [(700, 2, 1)], misalign=True),
    "simt_rows_p1": C(256, 256, [(300, 1, 1), (100, 2, 1)], impl=3, gelu=True),
    "simt_impl1": C(256, 256, [(700, 3, 1)], impl=1),
    # more than 64 groups: disjoint rows on the tensor cores, overlapping RTE-like groups on SIMT
    "g70_tc": C(64, 64, [(17 + 5 * i, 1, int(i % 3 != 1)) for i in range(70)]),
    "g70_rte": C(64, 64, [(240, 2, 0)] * 70, layout="rte"),
}
GAP, TAIL = 3, 5                   # uncovered A rows before every non-empty group, and past the last one


def build_table(c):
    """groups, cblocks, rows of A (TAIL past the end of the last group), end of the last group, W rows, out_elems."""
    groups, cblocks = [], []
    a0 = w0 = off = 0
    for m, ncb, has_b in c.spec:
        first = len(cblocks)
        if c.layout == "rte":
            row0 = 0
        else:
            if m:
                a0 += GAP
            row0 = a0
            a0 += m
        shift = 4 if c.misalign else 0
        if c.layout == "single":
            for _ in range(ncb):
                cblocks.append((off + shift, c.width))
                off += m * c.width + 32
        else:
            cblocks.append((off + shift, c.width))
            off += m * c.width + 32
            j = 1
            while j < ncb:
                pair = min(2, ncb - j)
                for q in range(pair):
                    cblocks.append((off + q * c.width + shift, 2 * c.width))
                off += m * 2 * c.width + 32
                j += pair
        off = -(-off // 32) * 32
        groups.append((row0, m, 0 if c.share_w else w0, ncb, first, has_b))
        if not c.share_w:
            w0 += ncb * c.width
    w_rows = max(g[2] + g[3] * c.width for g in groups)
    end = max((g[0] + g[1] for g in groups if g[1]), default=0)
    return groups, cblocks, end + TAIL, end, w_rows, off + 64


def case_instance(name, det, sms=H100_SMS):
    c = CASES[name]
    groups, cblocks = build_table(c)[:2]
    return bwd_instance(c.K, c.width, groups, cblocks, c.K + c.lda_pad, c.impl, c.dsplit, c.asplit, det, sms)


def test_case_list_reaches_every_instance():
    """CASES x {atomic, deterministic} reach the 18 tensor-core kernels, the four SIMT kernels, both split kernels,
    every reason for the SIMT path, and deterministic tasks of three or more dW chunks on both paths; the benchmark
    layers are among the cases."""
    inst = {(n, det): case_instance(n, det) for n in CASES for det in (False, True)}
    kernels = set().union(*(i.kernels for i in inst.values()))
    tc = {(k, tn, p) for k in ("k_lin_dx_tc", "k_lin_dw_tc", "k_lin_dw_tc_det") for tn in (64, 128, 256) for p in (3, 1)}
    simt = {(k,) for k in ("k_lin_dx_simt", "k_lin_dw_simt", "k_lin_dx_simt_det", "k_lin_dw_simt_det")}
    split = {("k_split_colsum",), ("k_split_colsum_det",)}
    assert kernels == tc | simt | split, sorted((tc | simt | split) - kernels)
    reasons = {i.reason for i in inst.values()} - {None}
    assert reasons == {"width % 8", "K % 16", "K < 64", "width < 16", "lda != K", "overlap", "align", "rows < 512",
                       "impl 1"}, reasons
    assert any(i.tc and i.dw_chunks >= 3 for (n, det), i in inst.items() if det)
    assert any(not i.tc and i.dw_chunks >= 3 for (n, det), i in inst.items() if det)
    for name, K in (("c2c4", 256), ("c3", 400), ("c5", 128)):
        c = CASES[name]
        assert c.K == c.width == K and inst[(name, False)].tc
    assert inst[("c3", False)].tile_n == 64 and -(-400 // 64) == 7 and 400 - 3 * BM == 16
    assert inst[("k80", False)].tile_n == 128 and inst[("k80", False)].tc
    rows = {m for c in CASES.values() for m, _, _ in c.spec}
    assert {0, 1, 63, 64, 65, 127, 129} <= rows and max(rows) > 3000
    assert {c.width for c in CASES.values() if c.K >= 64} >= {16, 24, 40, 1040}
    assert all(inst[(n, False)].tc for n in ("w16", "w24_p1", "w40", "w1040"))
    assert {c.layout for c in CASES.values()} == {"pairs", "single", "rte"}
    assert inst[("simt_k1169", False)].reason == "K % 16"
    assert CASES["simt_rte"].layout == "rte" and inst[("simt_rte", False)].reason == "overlap"
    assert len(CASES["g70_tc"].spec) > 64 and inst[("g70_tc", False)].tc
    assert len(CASES["g70_rte"].spec) > 64 and inst[("g70_rte", False)].reason == "overlap"


@pytest.mark.parametrize("n_groups", [65, 200])
@pytest.mark.parametrize("fn", ["hgt_typed_linear_bwd_workspace_bytes", "hgt_typed_linear_bwd_det_workspace_bytes"])
@pytest.mark.parametrize("K,width,overlap", [(64, 64, False), (64, 64, True), (48, 20, False)])
def test_workspace_accepts_more_than_64_groups(fn, n_groups, K, width, overlap):
    """Both backward workspace queries take any number of groups, and the workspace grows with the table."""
    sizes = []
    for n in (n_groups, 2 * n_groups):
        g = np.zeros(n, dtype=_lib.LIN_GROUP_DTYPE)
        c = np.zeros(n, dtype=_lib.LIN_CBLOCK_DTYPE)
        for i in range(n):
            g[i] = (0 if overlap else 600 * i, 600, i * width, 1, i, 1)
            c[i] = (i * 600 * width, width)
        b = ctypes.c_size_t()
        _lib.call(fn, g.ctypes.data, n, c.ctypes.data, K, width, K, n * 600 * width, 0, 0, 0, ctypes.byref(b))
        sizes.append(b.value)
    assert 0 < sizes[0] < sizes[1]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every case against float64

def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rne(t):
    return t.detach().to(BF16).double().cpu()


class Inputs:
    """Seeded operands of one case on the device: dout (flat), X (the layer input; A = gelu(X) when gelu), A in fp32
    with row stride lda, the producers' bf16 splits, W, the prefills of dW / db / accumulated dA, and the packed table."""

    def __init__(self, name):
        from pyhgt_b200 import plan as P
        c = self.c = CASES[name]
        dev = _dev()
        self.groups, self.cblocks, self.rows, self.end, self.w_rows, self.out_elems = build_table(c)
        self.tab = P._pack_groups(self.groups, self.cblocks, dev)
        self.K, self.lda = c.K, c.K + c.lda_pad
        gen = torch.Generator().manual_seed(sum(map(ord, name)))
        self.dout = torch.randn(self.out_elems, generator=gen).to(dev)
        self.X = torch.randn(self.rows, self.lda, generator=gen).to(dev)
        self.W = (torch.randn(self.w_rows, c.K, generator=gen) / math.sqrt(c.K)).to(dev)
        self.dW0 = torch.randn(self.w_rows, c.K, generator=gen).to(dev)
        self.db0 = torch.randn(self.w_rows, generator=gen).to(dev)
        self.dA0 = torch.randn(self.rows, c.K, generator=gen).to(dev)
        K, st = c.K, _st()
        self.A = self.X
        if c.gelu:
            assert c.lda_pad == 0
            self.A = torch.empty_like(self.X)
            _lib.call("hgt_act_split", self.X.data_ptr(), K, self.rows, K, 1, self.A.data_ptr(), None, None, st)
        self.a_hi = self.a_lo = self.d_hi = self.d_lo = None
        one = c.impl == 3
        if c.asplit:
            self.a_hi = torch.empty(self.rows, K, dtype=BF16, device=dev)
            self.a_lo = None if one else torch.empty(self.rows, K, dtype=BF16, device=dev)
            _lib.call("hgt_act_split", self.X.data_ptr(), K, self.rows, K, int(c.gelu), None, self.a_hi.data_ptr(),
                      _lib.ptr(self.a_lo), st)
        if c.dsplit:
            assert self.out_elems % 8 == 0
            self.d_hi = torch.empty(self.out_elems, dtype=BF16, device=dev)
            self.d_lo = None if one else torch.empty(self.out_elems, dtype=BF16, device=dev)
            _lib.call("hgt_act_split", self.dout.data_ptr(), self.out_elems, 1, self.out_elems, 0, None,
                      self.d_hi.data_ptr(), _lib.ptr(self.d_lo), st)

    def call(self, det, dA=True, acc=False, dW=True, db=True):
        """One backward call: returns (dA, dW, db), each None when not asked for.  dA starts NaN (random with acc),
        dW and db start at their prefills."""
        c, dev = self.c, _dev()
        g_dev, g_host, n_g, _ = self.tab
        fn = "hgt_typed_linear_bwd_det" if det else "hgt_typed_linear_bwd"
        a_out = (self.dA0.clone() if acc else torch.full((self.rows, c.K), float("nan"), device=dev)) if dA else None
        w_out = self.dW0.clone() if dW else None
        b_out = self.db0.clone() if db else None
        wsb = ctypes.c_size_t()
        _lib.call(fn + "_workspace_bytes", g_host.ctypes.data, n_g, self.tab.c_host.ctypes.data, c.K, c.width,
                  self.lda, self.out_elems, int(c.dsplit), int(c.asplit), c.impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        _lib.call(fn, None if c.dsplit else self.dout.data_ptr(), _lib.ptr(self.d_hi), _lib.ptr(self.d_lo),
                  self.out_elems, self.A.data_ptr(), self.lda, _lib.ptr(self.a_hi), _lib.ptr(self.a_lo),
                  self.W.data_ptr(), c.K, c.width, g_dev.data_ptr(), g_host.ctypes.data, n_g,
                  self.tab.c_host.ctypes.data, _lib.ptr(a_out), int(acc), self.X.data_ptr() if c.gelu else None,
                  _lib.ptr(w_out), _lib.ptr(b_out), c.impl, ws.data_ptr(), ws.numel(), _st())
        torch.cuda.synchronize()
        return a_out, w_out, b_out


def _gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def reference(inp, P):
    """float64 autograd of sum_blocks sum(dout * (act(X) W^T + b)) over the column-block table, with the operands the
    kernel multiplies (bf16-rounded at P = 1), and the elementwise scales of dA, dW and db (to be multiplied by TOL[P]).  db sums the fp32 dout
    (also at P = 1); groups without bias add nothing to it."""
    c, K, width = inp.c, inp.K, inp.c.width
    rnd = _rne if P == 1 else (lambda t: t.detach().double().cpu())
    d64 = inp.dout.double().cpu()
    dv, Wv = rnd(inp.dout), rnd(inp.W).requires_grad_(True)
    X = inp.X.double().cpu()[:, :K].requires_grad_(True)
    A_used = rnd(inp.A[:, :K])                 # the A the kernel multiplies: fp32 act(X) (its split, or rounded)
    act = _gelu64(X) if c.gelu else X
    A_st = act + (A_used - act).detach()       # value A_used, derivative act'(X)
    b = torch.zeros(inp.w_rows, dtype=torch.float64, requires_grad=True)
    loss = 0
    sc_dA = torch.zeros(inp.rows, K, dtype=torch.float64)
    sc_dW = torch.zeros(inp.w_rows, K, dtype=torch.float64)
    sc_db = torch.zeros(inp.w_rows, dtype=torch.float64)
    for a0, m, w0, ncb, cb0, has_b in inp.groups:
        for j in range(ncb):
            off, ld = inp.cblocks[cb0 + j]
            i = off + torch.arange(m)[:, None] * ld + torch.arange(width)[None]
            wr = slice(w0 + j * width, w0 + (j + 1) * width)
            y = A_st[a0:a0 + m] @ Wv[wr].T
            loss = loss + (dv[i] * y).sum()
            sc_dA[a0:a0 + m] += dv[i].abs() @ Wv[wr].detach().abs()
            sc_dW[wr] += dv[i].abs().T @ A_used[a0:a0 + m].abs()
            if has_b:
                loss = loss + (d64[i] * b[wr]).sum()
                sc_db[wr] += d64[i].abs().sum(0)
    loss.backward()
    ref_dA = X.grad if X.grad is not None else torch.zeros(inp.rows, K, dtype=torch.float64)
    ref_dW = Wv.grad if Wv.grad is not None else torch.zeros(inp.w_rows, K, dtype=torch.float64)
    ref_db = b.grad if b.grad is not None else torch.zeros(inp.w_rows, dtype=torch.float64)
    bound_dA = sc_dA
    if c.gelu:
        # gelu'(X) is evaluated in fp32 (erff, __expf): an absolute error of ~1e-6 on a factor that crosses zero
        xx = X.detach()
        gg = 0.5 * (1 + torch.erf(xx / math.sqrt(2))) + xx * torch.exp(-0.5 * xx * xx) / math.sqrt(2 * math.pi)
        bound_dA = sc_dA * gg.abs() + 1e-6 / TOL[P] * sc_dA
    return ref_dA, ref_dW, ref_db, bound_dA, sc_dW, sc_db


def _within(got, ref, scale, prefill, tol, what):
    """|got - (prefill + ref)| <= tol * (scale + |prefill|) everywhere (prefill None: 0); returns the worst ratio."""
    got = got.double().cpu()
    want = ref if prefill is None else ref + prefill.double().cpu()
    bound = tol * (scale + (0 if prefill is None else prefill.double().cpu().abs())) + 1e-30
    assert torch.isfinite(got).all(), "%s: non-finite values" % what
    ratio = ((got - want).abs() / bound).max().item()
    assert ratio <= 1.0, "%s: max |err| / bound = %.3g (tol %.1g)" % (what, ratio, tol)
    return ratio * tol


def _check_dA(inp, dA, ref, bound, tol, acc, what):
    """Covered rows: the gradient (+ the prefill with acc); rows between / before groups: 0 (the prefill with acc);
    rows past the last group: untouched (NaN, or the prefill)."""
    covered = torch.zeros(inp.rows, dtype=torch.bool)
    for a0, m, *_ in inp.groups:
        covered[a0:a0 + m] = True
    dA = dA.cpu()
    pre = inp.dA0.cpu()
    if acc:
        assert torch.equal(dA[~covered], pre[~covered]), "%s: uncovered rows of an accumulated dA changed" % what
    else:
        gap = ~covered
        gap[inp.end:] = False
        assert (dA[gap] == 0).all(), "%s: rows between groups are not zero" % what
        assert torch.isnan(dA[inp.end:]).all(), "%s: rows past the last group were written" % what
    return _within(dA[covered], ref[covered], bound[covered], pre[covered] if acc else None, tol, what)


def _check_db(inp, db, ref, scale, tol, what):
    """db rows of has_bias groups: prefill + gradient; every other row (all rows with a pre-split dout): the prefill."""
    biased = torch.zeros(inp.w_rows, dtype=torch.bool)
    if not inp.c.dsplit:
        for a0, m, w0, ncb, cb0, has_b in inp.groups:
            if has_b:
                biased[w0:w0 + ncb * inp.c.width] = True
    db, pre = db.cpu(), inp.db0.cpu()
    assert torch.equal(db[~biased], pre[~biased]), "%s: db rows without bias changed" % what
    if biased.any():
        return _within(db[biased], ref[biased], scale[biased], pre[biased], tol, what)
    return 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_linear_bwd_instance_matches_fp64(name, det):
    """dA, dW and db of one case against float64, from sentinel-filled outputs; accumulate_dA; each output NULL in
    turn; the deterministic entry point twice, bitwise equal."""
    inp = Inputs(name)
    c = inp.c
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    inst = bwd_instance(c.K, c.width, inp.groups, inp.cblocks, inp.lda, c.impl, c.dsplit, c.asplit, det, sms)
    tol = TOL[inst.P]
    ref_dA, ref_dW, ref_db, b_dA, s_dW, s_db = reference(inp, inst.P)
    tag = "%s %s (%s)" % (name, "det" if det else "atomic", "tc BN %d P %d" % (inst.tile_n, inst.P) if inst.tc
                          else "simt: " + inst.reason)

    full = inp.call(det)
    worst = [_check_dA(inp, full[0], ref_dA, b_dA, tol, False, tag + " dA"),
             _within(full[1], ref_dW, s_dW, inp.dW0, tol, tag + " dW"),
             _check_db(inp, full[2], ref_db, s_db, tol, tag + " db")]
    print("\n%s: worst |err| / scale dA %.2e dW %.2e db %.2e" % (tag, *worst))
    if det:
        again = inp.call(det)
        for x, y, what in zip(full, again, ("dA", "dW", "db")):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "%s %s: two runs differ" % (tag, what)

    acc = inp.call(det, acc=True)
    _check_dA(inp, acc[0], ref_dA, b_dA, tol, True, tag + " accumulated dA")
    _within(acc[1], ref_dW, s_dW, inp.dW0, tol, tag + " dW (accumulate_dA)")

    for skip in ("dA", "dW", "db"):
        out = inp.call(det, dA=skip != "dA", dW=skip != "dW", db=skip != "db")
        what = "%s, %s NULL:" % (tag, skip)
        if skip != "dA":
            _check_dA(inp, out[0], ref_dA, b_dA, tol, False, what + " dA")
        if skip != "dW":
            _within(out[1], ref_dW, s_dW, inp.dW0, tol, what + " dW")
        if skip != "db":
            _check_db(inp, out[2], ref_db, s_db, tol, what + " db")
        if det:
            for x, y, nm in zip(out, full, ("dA", "dW", "db")):
                if x is not None:
                    assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "%s %s differs" % (what, nm)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: a training step with more than 64 <source type, relation> pairs

@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_rte_layer_with_more_than_64_pairs_matches_fp64(det, monkeypatch):
    """HGTConv(use_RTE=True) on 9 types x 8 relations: its RTE projection has one group per present pair (more than 64).
    One training step against float64 autograd through the oracle port, atomic and deterministic; the deterministic
    step repeats bitwise."""
    import pyhgt_b200
    from pyhgt_b200 import plan as P, synth
    from tests.test_gpu_deterministic import _assert_bitwise, _deterministic
    from tests.test_gpu_grad_parity import _compare_all, _f64_params, _native_layer, _oracle_layer, _perturb
    dev = _dev()
    monkeypatch.setattr(pyhgt_b200.HGTConv, "keep_att", False)
    T, R, d, H = 9, 8, 64, 4
    g = synth.make_random(3000, 24000, T, R, seed=65, isolated_frac=0.1, self_loops=40)
    plan = P.get_plan(g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev), T, R)
    assert plan.n_pairs > 64, plan.n_pairs
    torch.manual_seed(66)
    m = _perturb(pyhgt_b200.HGTConv(d, d, T, R, H, 0.0, True, True), 67)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(68))
    w = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(69))
    params = _f64_params(m)
    xr = x.double().requires_grad_(True)
    out = _oracle_layer(params, xr, g, m)
    (out * w.double()).sum().backward()
    ref = (out.detach(), xr.grad, {k: v.grad for k, v in params.items()})
    state = m.state_dict()

    def step():
        layer = pyhgt_b200.HGTConv(d, d, T, R, H, 0.0, True, True)
        layer.load_state_dict(state)
        return _native_layer(layer.to(dev).train(), x, g, w, dev)

    with _deterministic(det):
        a = step()
        if det:
            _assert_bitwise(a, step(), "RTE, %d pairs" % plan.n_pairs)
    _compare_all("RTE, %d pairs, deterministic %s" % (plan.n_pairs, det), a, ref, (4e-5, 2.5e-4))
