"""Every compiled instance of the forward typed GEMM (csrc/linear_tc.cu, and the SIMT kernel in csrc/linear.cu) against
float64 on the same tables.

hgt_typed_linear / _bf16 / _t24 / _bf16a and hgt_typed_linear_presplit / _presplit_bf16 / _presplit_t24 (with or without
a_lo) run either the fp32 SIMT kernel k_typed_linear_simt<AT, OutT> or the tensor-core kernel
k_typed_linear_tc<BN, OutT, P, KB, AF>, behind pre-passes (the bf16 split of W, of A into the workspace at 64-column
tiles or into private memory for an fp32 A that TMA cannot load, the zero-padding copy of a bf16 A, the output tensor
maps at 128 / 256-column tiles), in launches of at most 64 groups.  `fwd_instance` restates that choice (typed_linear,
hgt_typed_linear_tc_supported, splits_a_first, a_fp32_loadable, run_fwd, hgt_typed_linear_tc_bf16a), and
test_case_list_reaches_every_instance (no GPU needed) checks that CASES, with HGT_TC_P1_KB unset, 32 and 64, reach all 45
tensor-core instances, the four SIMT instances, every pre-pass, both epilogues (TMA tensor stores and staged stores) for
every output type at 128 and 256 columns, and a launch in which one CTA alternates between the two.

References (elementwise, as in test_gpu_linear_bwd_instances.py):
  three products, bf16 A (P = 2) and fp32 SIMT   float64 of the exact operands, |err| <= TOL[P] (|a| |w| + |b|)
  one product                                    float64 of the bf16-rounded A and W, |err| <= ACC_TOL (|a| |w| + |b|)
  bf16 output                                    bitwise the RNE of the fp32 entry point's output
  24-bit output                                  bitwise round_words of the fp32 output, decoded within the bound plus
                                                 half a 24-bit ulp; fp32 blocks of a mixed call bitwise the fp32 output
Every output starts from a sentinel (a NaN bit pattern, or the byte 0xA5 in the 24-bit planes) that every element outside
the column blocks keeps: gaps between blocks, ld padding, the masked columns of a tile, and the elements around the
buffer.  A's padding columns and the rows between groups hold NaN, so reading one shows.  Each call launches as many
kernels (_lib.kernel_launches) as the restatement predicts.  Cross-checks that must hold bitwise: an fp32 A
that TMA loads (AF: split in shared memory) against the same A split first by k_split_bf16 (the presplit kernel), and the
two k-blocks (32 and 64) of the one-product kernel, run in child processes under HGT_TC_P1_KB because the library reads
the switch once per process.  The k-blocks run the same 16-wide wgmma steps in the same k order; the longer k-block only
adds more zero-filled steps past Kp.

Worst |err| / (|a| |w| + |b|) measured on an H100 SXM (132 SMs), against the bounds 5e-5 / 1e-5: 6.6e-6 with three
products, 2.4e-6 with a bf16 A (P = 2), 2.8e-7 with one product (against the rounded operands) and 3.3e-7 on the fp32
SIMT kernel.  The two one-product k-blocks wrote the same bits in every case there.
"""
import ctypes
import math
import os
import subprocess
import sys
from collections import namedtuple

import pytest
import torch

from pyhgt_b200 import _lib
from tests.test_gpu_linear_bwd_instances import GAP, H100_SMS, TAIL, TOL, pick_tile_n

BF16 = torch.bfloat16
BM = 128                           # tile rows of both kernels
SIMT_BN = 64                       # tile columns of the SIMT kernel
MAX_GROUPS = 64                    # groups per launch
ACC_TOL = 1e-5                     # test_gpu_matmul_precision.ACC_TOL: one product
FWD_TOL = {3: TOL[3], 2: TOL[3], 1: ACC_TOL, None: TOL[None]}    # keyed by bf16 products; None: fp32 SIMT
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_KINDS = ("fp32", "bf16", "t24")


# ---------------------------------------------------------------------------------------------------------------------
# the kernel-selection rule, restated

def fwd_bk(bn):
    return 64 if bn == 64 else 32


def kb_env_of(value):
    """The library's reading of HGT_TC_P1_KB: "32..." -> 32, "64..." -> 64, anything else (or unset) -> None."""
    if value and value[:2] == "32":
        return 32
    if value and value[:2] == "64":
        return 64
    return None


def out_kind(entry):
    return "bf16" if entry.endswith("_bf16") else "t24" if entry.endswith("_t24") else "fp32"


def _t24_bytes(L, ld):
    """Byte of the hi (u16) and of the lo (u8) plane of logical 24-bit offset L in a table of rows of ld elements."""
    col = L % ld
    return 3 * (L - col) + 2 * col, 3 * (L - col) + 2 * ld + col


def _epilogue(kind, off, ld, t24_off):
    """(plane, mode) of a column block at 128 / 256-column tiles; out / out32 / out24 bases are 16-byte aligned."""
    if kind == "t24" and off < t24_off:
        return "t24/fp32", "tma" if (off * 4) % 16 == 0 and (ld * 4) % 16 == 0 else "staged"
    if kind == "t24":
        hi, lo = _t24_bytes(off - t24_off, ld)
        return "t24", "tma" if (hi | lo | 3 * ld) % 16 == 0 else "staged"
    size = 2 if kind == "bf16" else 4
    return kind, "tma" if (off * size) % 16 == 0 and (ld * size) % 16 == 0 else "staged"


def _alternates(modes):
    """Some tile stored by TMA, a later one staged, and a later one by TMA again."""
    seen = 0
    for m in modes:
        if m == ("tma", "staged", "tma")[seen]:
            seen += 1
            if seen == 3:
                return True
    return False


# path: "simt" or "tc"; P: bf16 products (None on SIMT); launches: kernel keys in launch order; epilogues:
# {(plane, BN, "tma" | "staged")}; alternates: a CTA of some launch stores TMA, staged and TMA tiles in that order
Instance = namedtuple("Instance", "path P launches epilogues alternates")


def fwd_instance(entry, impl, K, width, lda, a_aligned, groups, cblocks, kb_env, a_lo=True, t24_off=0, sms=H100_SMS):
    """What one call does.  entry: the C entry point; impl: 0..3 (ignored by the presplit entry points, which run three
    products with a_lo and one without); a_aligned: A's base is 16-byte aligned; groups: (a_row0, m, w_row0, n_cblocks,
    cb_first, has_bias); cblocks: (out_off, ld); kb_env: HGT_TC_P1_KB as the library reads it (None, 32, 64)."""
    kind = out_kind(entry)
    presplit = "presplit" in entry
    bf16a = entry.endswith("_bf16a")
    at = "bf16" if bf16a else "fp32"
    tc_ok = width % 16 == 0 and width > 0 and K >= 64
    if presplit:
        assert K % 8 == 0 and tc_ok
        tc, P = True, 3 if a_lo else 1
    else:
        if impl == 0:
            impl = 2 if tc_ok else 1
        if impl == 3 and not tc_ok:
            impl = 1                              # fp32 SIMT, not one bf16 product
        assert impl != 2 or tc_ok
        tc = impl in (2, 3)
        P = (1 if impl == 3 else 2 if bf16a else 3) if tc else None
    launches, epilogues, alternates = [], set(), False
    for c0 in range(0, len(groups), MAX_GROUPS):
        chunk = groups[c0:c0 + MAX_GROUPS]
        if not tc:
            if sum(-(-m // BM) * ncb * -(-width // SIMT_BN) for _, m, _, ncb, _, _ in chunk):
                launches.append(("k_typed_linear_simt", at, kind))
            continue
        bn = pick_tile_n(width)
        a_rows = max(a0 + m for a0, m, *_ in chunk)
        launches.append(("k_split_bf16", "W"))
        af = False
        if presplit:
            pass
        elif bf16a:
            if not (a_aligned and lda % 8 == 0 and K % 8 == 0):
                if a_rows == 0:
                    continue
                launches.append(("k_pad_bf16",))
        elif bn == 64:
            if a_rows == 0:
                continue
            launches.append(("k_split_bf16", "A"))
        elif a_aligned and lda % 4 == 0:
            af = True
        else:
            if a_rows == 0:
                continue
            launches.append(("k_split_bf16", "A private"))
        n_tn = -(-width // bn)
        tiles = []
        for _, m, _, ncb, cb0, _ in chunk:
            modes = [_epilogue(kind, *cblocks[cb0 + j], t24_off) for j in range(ncb)]
            for _ in range(-(-m // BM)):
                for j in range(ncb):
                    tiles += [modes[j]] * n_tn
        if not tiles:
            continue
        kb = fwd_bk(bn)
        if P == 1 and bn != 64:
            kb = kb_env or (32 if af else 64)
        if bn != 64:
            launches.append(("k_out_maps", kind))
            epilogues |= {(plane, bn, mode) for plane, mode in tiles}
            grid = min(len(tiles), sms)
            alternates |= any(_alternates([m for _, m in tiles[b::grid]]) for b in range(grid))
        launches.append(("k_typed_linear_tc", bn, kind, P, kb, af))
    return Instance("tc" if tc else "simt", P, launches, epilogues, alternates)


# ---------------------------------------------------------------------------------------------------------------------
# cases

Case = namedtuple("Case", "a impl K width spec layout pad shifts lda a_off share_w bias t24")


def C(a, K, width, spec, impl=0, layout="proj", pad=0, shifts=(0,), lda=None, a_off=0, share_w=False, bias=True,
      t24="all"):
    """a: "fp32" (hgt_typed_linear[_bf16|_t24]), "presplit" / "presplit1" (hgt_typed_linear_presplit[_bf16|_t24] with
    and without a_lo) or "bf16" (hgt_typed_linear_bf16a).  spec: [(rows, column blocks, has_bias)].  layout "proj": a
    group's first column block in rows of ld = width + pad, the others two by two in rows of ld = 2 width + pad (the
    projection table); "single": every block in its own rows of ld = width + pad; "rte": the pairs layout, every group
    reading rows 0..rows of the same A (the RTE tables' overlapping groups).  shifts: the blocks of the i-th region
    start shifts[i % len] elements into their rows (<= pad).  lda (default K), a_off: A's row stride and the elements
    between the allocation and A.  bias False: bias = NULL.  t24 "mixed": the first group's blocks are fp32 blocks (before
    t24_off) of the 24-bit call."""
    assert all(s <= pad for s in shifts)
    return Case(a, impl, K, width, spec, layout, pad, shifts, K if lda is None else lda, a_off, share_w, bias, t24)


def _g70(i):
    return (17 + 5 * i, 1, int(i % 3 != 1))


CASES = {
    # the benchmark layer shapes: c2 (d = 256), c3 (d = 400: 64-column tiles, the last one 16 columns wide), c5 (d = 128)
    "c2": C("fp32", 256, 256, [(3001, 3, 1), (129, 1, 0), (0, 1, 1), (1, 2, 1)], t24="mixed"),
    "c2_p1": C("fp32", 256, 256, [(65, 3, 1), (3100, 1, 1), (127, 2, 0)], impl=3, pad=8),
    "c3": C("fp32", 80, 400, [(900, 3, 1), (65, 1, 0), (0, 1, 1), (64, 2, 1)], t24="mixed"),
    "c3_p1": C("fp32", 72, 400, [(600, 3, 1), (63, 1, 1)], impl=3, layout="single", pad=8, shifts=(0, 3)),
    "c5_presplit": C("presplit", 128, 128, [(63, 1, 1), (64, 2, 0), (127, 1, 1), (300, 3, 1)], layout="single", pad=16,
                     shifts=(0, 1)),
    # column blocks that end inside a tile (80 of 128 columns); aligned and misaligned blocks alternate in the tiles of
    # one CTA (group 0: 275 tiles over 132 CTAs)
    "w80_alt": C("fp32", 72, 80, [(7000, 5, 1), (129, 5, 0)], impl=2, layout="single", pad=16, shifts=(0, 0, 1, 2, 0),
                 t24="mixed"),
    "w256_alt": C("fp32", 64, 256, [(4000, 3, 1), (128, 2, 1)], layout="single", pad=16, shifts=(0, 1, 2)),
    # K with a partial last k-block (72, 80) or Kp > K (129, 1169); fp32 A with lda > K (AF), lda % 4 != 0 or a base 4
    # bytes off 16-byte alignment (split first)
    "k129_af": C("fp32", 129, 128, [(300, 3, 1), (64, 1, 1)], lda=132, pad=8, t24="mixed"),
    "k129": C("fp32", 129, 256, [(200, 3, 1), (1, 1, 0)], pad=16, shifts=(0, 1)),
    "k1169_af": C("fp32", 1169, 256, [(129, 2, 1), (63, 1, 1)], lda=1172, layout="single"),
    "k129_p1_af": C("fp32", 129, 128, [(300, 3, 1), (127, 1, 0)], impl=3, lda=132, pad=16, shifts=(0, 1), t24="mixed"),
    "k1169_p1": C("fp32", 1169, 256, [(200, 1, 1), (65, 2, 1)], impl=3, pad=8),
    "a_off": C("fp32", 64, 128, [(300, 3, 1), (128, 1, 1)], a_off=1, lda=68, pad=8),
    "a_off_p1": C("fp32", 80, 256, [(257, 2, 1)], impl=3, a_off=1, t24="mixed"),
    "k72_lda": C("fp32", 72, 64, [(300, 2, 1), (129, 1, 1)], lda=73, t24="mixed"),
    "bias_null": C("fp32", 80, 256, [(200, 3, 1), (129, 1, 1)], bias=False, pad=16, shifts=(0, 1)),
    # groups sharing W rows, and overlapping A rows (RTE layout) on the tensor cores
    "shared_w": C("fp32", 64, 128, [(700, 2, 1), (300, 2, 1)], share_w=True, t24="mixed"),
    "rte_tc": C("fp32", 64, 128, [(240, 2, 0)] * 5 + [(240, 2, 1)], layout="rte"),
    "rte_tc_p1": C("fp32", 64, 256, [(240, 2, 1)] * 4, impl=3, layout="rte", pad=8, t24="mixed"),
    # presplit A, with a_lo (P = 3) and without (P = 1)
    "presplit_w256": C("presplit", 72, 256, [(300, 3, 1), (129, 1, 0)], pad=8, shifts=(0, 1), t24="mixed"),
    "presplit_w400": C("presplit", 80, 400, [(333, 2, 1), (64, 1, 1)]),
    "presplit1_w128": C("presplit1", 64, 128, [(400, 3, 1), (65, 1, 1)], pad=16, shifts=(0, 1), t24="mixed"),
    "presplit1_w256": C("presplit1", 80, 256, [(300, 2, 1), (1, 1, 1)], layout="single", pad=8),
    "presplit1_w80": C("presplit1", 1168, 80, [(129, 2, 1)], pad=16, shifts=(0, 1), t24="mixed"),
    "presplit1_w64": C("presplit1", 64, 64, [(200, 2, 1), (37, 1, 0)]),
    # bf16 A: in place, lda % 8 != 0, K % 8 != 0, a base 2 bytes off; two products (P = 2) and one
    "bf16_w256": C("bf16", 64, 256, [(300, 3, 1), (129, 1, 0)]),
    "bf16_lda": C("bf16", 64, 128, [(300, 3, 1), (65, 1, 1)], lda=68),
    "bf16_k129": C("bf16", 129, 400, [(200, 2, 1), (63, 1, 1)]),
    "bf16_off": C("bf16", 80, 80, [(300, 2, 1)], a_off=1, pad=16, shifts=(0, 1)),
    "bf16_p1": C("bf16", 80, 256, [(300, 2, 1), (64, 1, 1)], impl=3, pad=16, shifts=(0, 1)),
    "bf16_p1_w128": C("bf16", 1168, 128, [(129, 2, 1)], impl=3),
    "bf16_p1_w64": C("bf16", 72, 64, [(200, 2, 1)], impl=3, lda=76),
    # fp32 SIMT: impl 1, K < 64, width % 16 != 0, and impl 3 falling back to fp32 (not one bf16 product)
    "simt_impl1": C("fp32", 256, 256, [(700, 3, 1), (0, 1, 1), (65, 1, 0)], impl=1, pad=8, t24="mixed"),
    "simt_k48": C("fp32", 48, 32, [(700, 2, 1)], lda=50, a_off=1),
    "simt_w40": C("fp32", 64, 40, [(300, 3, 1), (1, 1, 0)], pad=8, shifts=(0, 3), t24="mixed"),
    "simt_k48_p1": C("fp32", 48, 64, [(400, 2, 1)], impl=3),
    "simt_w20_p1": C("fp32", 129, 20, [(300, 2, 1)], impl=3, layout="single"),
    "simt_bf16": C("bf16", 64, 64, [(700, 2, 1), (64, 1, 0)], impl=1, lda=66, a_off=1),
    "simt_bf16_k40": C("bf16", 40, 128, [(300, 2, 1)], bias=False),
    # more than 64 groups: chunked launches on both paths, every output type
    "g70_tc": C("fp32", 64, 64, [_g70(i) for i in range(70)], t24="mixed"),
    "g70_w256": C("fp32", 64, 256, [_g70(i) for i in range(70)], impl=3, pad=8),
    "g70_presplit": C("presplit", 64, 128, [_g70(i) for i in range(70)], pad=16, shifts=(0, 1)),
    "g70_bf16": C("bf16", 64, 128, [_g70(i) for i in range(70)]),
    "g70_simt": C("fp32", 48, 40, [(240, 2, 0)] * 69 + [(240, 2, 1)], layout="rte", t24="mixed"),
}
GAP_ELEMS = 48                     # output elements between regions (sentinels)
HEAD = 64                          # sentinel elements (bytes for 24-bit planes) before and after each output


def build_table(c):
    """groups, cblocks, rows of A, t24_off, logical output size, W rows.  Regions start at multiples of their ld
    (counted from t24_off for the 24-bit groups), as the 24-bit row format needs."""
    groups, cblocks = [], []
    a0 = w0 = cur = t24_off = region = 0
    for gi, (m, ncb, has_b) in enumerate(c.spec):
        if c.t24 == "mixed" and gi == 1:
            t24_off = -(-(cur + GAP_ELEMS) // 16) * 16
            cur = t24_off
        base = t24_off
        if c.layout == "rte":
            row0 = 0
        else:
            if m:
                a0 += GAP
            row0, a0 = a0, a0 + m
        first = len(cblocks)
        if c.layout == "single":
            runs = [1] * ncb
        elif c.layout == "proj":
            runs = [1] + [2] * ((ncb - 1) // 2) + [1] * ((ncb - 1) % 2)
        else:
            runs = [2] * (ncb // 2) + [1] * (ncb % 2)
        for n in runs:
            ld = n * c.width + c.pad
            start = base + -(-(cur + GAP_ELEMS - base) // ld) * ld
            s = c.shifts[region % len(c.shifts)]
            region += 1
            cblocks += [(start + q * c.width + s, ld) for q in range(n)]
            cur = start + m * ld
        groups.append((row0, m, 0 if c.share_w else w0, ncb, first, has_b))
        if not c.share_w:
            w0 += ncb * c.width
    w_rows = max(g[2] + g[3] * c.width for g in groups)
    end = max((g[0] + g[1] for g in groups if g[1]), default=0)
    return groups, cblocks, end + TAIL, t24_off, cur + GAP_ELEMS, w_rows


def entries(c):
    if c.a == "bf16":
        return ("hgt_typed_linear_bf16a",)
    pre = "hgt_typed_linear_presplit" if c.a.startswith("presplit") else "hgt_typed_linear"
    return (pre, pre + "_bf16", pre + "_t24")


def case_instance(name, entry, kb_env, a_off=None):
    c = CASES[name]
    groups, cblocks, _, t24_off, _, _ = build_table(c)
    a_off = c.a_off if a_off is None else a_off
    a_aligned = (a_off * (2 if c.a == "bf16" else 4)) % 16 == 0
    return fwd_instance(entry, c.impl, c.K, c.width, c.lda, a_aligned, groups, cblocks, kb_env, a_lo=c.a != "presplit1",
                        t24_off=t24_off if c.t24 == "mixed" else 0)


def _tc_key(bn, kind, P, kb, af):
    return ("k_typed_linear_tc", bn, kind, P, kb, af)


def test_case_list_reaches_every_instance():
    """CASES x HGT_TC_P1_KB in {unset, 32, 64} reach the 45 tensor-core instances, the four SIMT instances, every
    pre-pass, both epilogues for each output type (and for the fp32 blocks of a mixed 24-bit call) at 128 and 256
    columns, and a launch where aligned and misaligned blocks alternate in the tiles of one CTA."""
    inst = {(n, e, kb): case_instance(n, e, kb) for n in CASES for e in entries(CASES[n]) for kb in (None, 32, 64)}
    launched = {k for i in inst.values() for k in i.launches}
    kinds = OUT_KINDS
    tc = {_tc_key(64, k, 3, 64, False) for k in kinds}
    tc |= {_tc_key(bn, k, 3, 32, af) for bn in (128, 256) for k in kinds for af in (False, True)}
    tc |= {_tc_key(bn, "fp32", 2, fwd_bk(bn), False) for bn in (64, 128, 256)}
    tc |= {_tc_key(64, k, 1, 64, False) for k in kinds}
    tc |= {_tc_key(bn, k, 1, kb, af) for bn in (128, 256) for k in kinds for kb in (32, 64) for af in (False, True)}
    assert len(tc) == 45
    simt = {("k_typed_linear_simt", "fp32", k) for k in kinds} | {("k_typed_linear_simt", "bf16", "fp32")}
    pre = {("k_split_bf16", "W"), ("k_split_bf16", "A"), ("k_split_bf16", "A private"), ("k_pad_bf16",)}
    pre |= {("k_out_maps", k) for k in kinds}
    assert launched == tc | simt | pre, (sorted(map(str, (tc | simt | pre) - launched)),
                                         sorted(map(str, launched - (tc | simt | pre))))
    # the k-block variants that only the switch reaches
    default = {k for (n, e, kb), i in inst.items() if kb is None for k in i.launches}
    switch_only = {_tc_key(bn, k, 1, 64, True) for bn in (128, 256) for k in kinds}
    switch_only |= {_tc_key(bn, k, 1, 32, False) for bn in (128, 256) for k in kinds}
    assert tc - default == switch_only
    epi = {e for i in inst.values() for e in i.epilogues}
    want = {(p, bn, m) for p in ("fp32", "bf16", "t24", "t24/fp32") for bn in (128, 256) for m in ("tma", "staged")}
    assert want <= epi, sorted(want - epi)
    assert any(i.alternates for i in inst.values())
    assert inst[("w80_alt", "hgt_typed_linear", None)].alternates
    # shapes, operands and layouts the issue of each path depends on
    rows = {m for c in CASES.values() for m, _, _ in c.spec}
    assert {0, 1, 63, 64, 65, 127, 128, 129} <= rows and max(rows) > 3000
    assert {pick_tile_n(c.width) for c in CASES.values()} == {64, 128, 256}
    assert {80, 400} <= {c.width for c in CASES.values()} and 400 - 6 * 64 == 16
    assert {64, 72, 80, 129, 1169} <= {c.K for c in CASES.values()}
    assert any(c.a == "fp32" and c.K == 129 and c.lda == 132 for c in CASES.values())
    assert any(c.a == "fp32" and c.a_off for c in CASES.values())
    assert any(c.a == "fp32" and c.lda % 4 for c in CASES.values())
    assert any(c.a == "fp32" and c.lda > c.K and c.lda % 4 == 0 and not c.a_off for c in CASES.values())
    bf = [c for c in CASES.values() if c.a == "bf16" and c.impl != 1 and c.K >= 64]
    assert any(c.lda % 8 == 0 and c.K % 8 == 0 and not c.a_off for c in bf)
    assert any(c.lda % 8 for c in bf) and any(c.K % 8 for c in bf) and any(c.a_off for c in bf)
    assert {c.layout for c in CASES.values()} == {"proj", "single", "rte"}
    assert any(c.share_w for c in CASES.values()) and any(not c.bias for c in CASES.values())
    assert any(m == 0 and 0 < i < len(c.spec) - 1 for c in CASES.values() for i, (m, _, _) in enumerate(c.spec))
    assert any(not hb for c in CASES.values() for _, _, hb in c.spec)
    assert {c.t24 for c in CASES.values() if c.a != "bf16"} == {"all", "mixed"}
    assert any(c.pad == 8 for c in CASES.values())
    # more than 64 groups on the tensor cores for every output type, and on SIMT
    big = [(n, e) for n, c in CASES.items() if len(c.spec) > MAX_GROUPS for e in entries(c)]
    assert {out_kind(e) for n, e in big if inst[(n, e, None)].path == "tc"} == set(kinds)
    assert {out_kind(e) for n, e in big if inst[(n, e, None)].path == "simt"} == set(kinds)
    # impl 3 where the tensor cores do not apply runs fp32 SIMT
    assert inst[("simt_k48_p1", "hgt_typed_linear", None)].P is None


def test_kb_switch_reading():
    assert [kb_env_of(v) for v in (None, "", "32", "64", "640", "3", "128")] == [None, None, 32, 64, 64, None, None]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every case against float64

SENT32 = 0x7FBADBAD                # NaN bit patterns no kernel writes
SENT16 = 0x7FBB
SENT8 = 0xA5


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.view({torch.float32: torch.int32, BF16: torch.int16}.get(t.dtype, t.dtype))


class Inputs:
    """Seeded operands of one case on the device (A with NaN in its padding columns and in the rows outside every group),
    the packed table and the float64 reference of every covered output element."""

    def __init__(self, name):
        from pyhgt_b200 import plan as P
        c = self.c = CASES[name]
        dev = _dev()
        self.groups, self.cblocks, self.rows, self.t24_off, self.out_elems, self.w_rows = build_table(c)
        if c.t24 != "mixed":
            self.t24_off = 0
        self.tab = P._pack_groups(self.groups, self.cblocks, dev)
        gen = torch.Generator().manual_seed(sum(map(ord, name)))
        K, lda = c.K, c.lda
        A = torch.full((self.rows, lda), float("nan"))
        covered = torch.zeros(self.rows, dtype=torch.bool)
        for a0, m, *_ in self.groups:
            covered[a0:a0 + m] = True
        A[covered, :K] = torch.randn(int(covered.sum()), K, generator=gen)
        if c.a == "bf16":
            A = A.to(BF16)
        self.A64 = A[:, :K].double()
        self.W = (torch.randn(self.w_rows, K, generator=gen) / math.sqrt(K))
        self.b = torch.randn(self.w_rows, generator=gen)
        flat = torch.cat([torch.zeros(c.a_off, dtype=A.dtype), A.reshape(-1), torch.zeros(8, dtype=A.dtype)])
        self.a_buf = flat.to(dev)
        self.a_ptr = self.a_buf.data_ptr() + c.a_off * A.element_size()
        self.W_dev, self.b_dev = self.W.to(dev), self.b.to(dev)
        self.hi = self.lo = None
        if c.a.startswith("presplit"):
            Ad = A.to(dev)
            self.hi = Ad.to(BF16)
            self.lo = (Ad - self.hi.float()).to(BF16) if c.a == "presplit" else None
        self._refs = {}

    def reference(self, P):
        """Flat output indices of the covered elements, their float64 values and elementwise scales (|a| |w| + |b|)
        with the operands the kernel multiplies (bf16-rounded at P = 1), and the ld of each element's block."""
        if P in self._refs:
            return self._refs[P]
        c = self.c
        rnd = (lambda t: t.to(BF16).double()) if P == 1 else (lambda t: t.double())
        A = self.A64 if P != 1 else self.A64.float().to(BF16).double()
        W = rnd(self.W)
        b = self.b.double() if c.bias else torch.zeros(self.w_rows, dtype=torch.float64)
        idx, ref, scale, lds = [], [], [], []
        for a0, m, w0, ncb, cb0, has_b in self.groups:
            if m == 0:
                continue
            Wg = W[w0:w0 + ncb * c.width]
            bg = b[w0:w0 + ncb * c.width] * has_b
            y = A[a0:a0 + m] @ Wg.T + bg
            s = A[a0:a0 + m].abs() @ Wg.abs().T + bg.abs()
            for j in range(ncb):
                off, ld = self.cblocks[cb0 + j]
                cols = slice(j * c.width, (j + 1) * c.width)
                idx.append((off + torch.arange(m)[:, None] * ld + torch.arange(c.width)[None]).reshape(-1))
                ref.append(y[:, cols].reshape(-1))
                scale.append(s[:, cols].reshape(-1))
                lds.append(torch.full((m * c.width,), ld, dtype=torch.int64))
        cat = (lambda x, dt: torch.cat(x) if x else torch.zeros(0, dtype=dt))
        r = self._refs[P] = (cat(idx, torch.int64), cat(ref, torch.float64), cat(scale, torch.float64),
                             cat(lds, torch.int64))
        return r

    def call(self, entry, a_ptr=None):
        """One call from sentinel-filled outputs.  Returns (raw buffer(s) with HEAD sentinels each side, the kernel keys
        the library's kernel launches of the call)."""
        c, dev = self.c, _dev()
        g_dev, g_host, n_g, c_dev = self.tab
        kind = out_kind(entry)
        n = self.out_elems
        out32 = out16 = out24 = None
        if kind == "fp32":
            out32 = torch.full((n + 2 * HEAD,), SENT32, dtype=torch.int32, device=dev).view(torch.float32)
        elif kind == "bf16":
            out16 = torch.full((n + 2 * HEAD,), SENT16, dtype=torch.int16, device=dev).view(BF16)
        else:
            out32 = torch.full((self.t24_off + 2 * HEAD,), SENT32, dtype=torch.int32, device=dev).view(torch.float32)
            out24 = torch.full((3 * (n - self.t24_off) + 2 * HEAD,), SENT8, dtype=torch.uint8, device=dev)
        for t in (out32, out16, out24):
            assert t is None or t.data_ptr() % 256 == 0
        at = (lambda t: None if t is None else t.data_ptr() + HEAD * t.element_size())
        wsb = ctypes.c_size_t()
        if c.a.startswith("presplit"):
            _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, c.K, c.width,
                      ctypes.byref(wsb))
        else:
            _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, c.K, c.width, c.impl, ctypes.byref(wsb))
        ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
        bias = self.b_dev.data_ptr() if c.bias else None
        if c.a.startswith("presplit"):
            head = (self.hi.data_ptr(), _lib.ptr(self.lo))
            outs = {"fp32": (at(out32),), "bf16": (at(out16),), "t24": (at(out32), self.t24_off, at(out24))}[kind]
            args = head + (self.W_dev.data_ptr(), bias, c.K, c.width, g_dev.data_ptr(), g_host.ctypes.data, n_g,
                           c_dev.data_ptr()) + outs + (ws.data_ptr(), ws.numel(), _st())
        else:
            outs = {"fp32": (at(out32),), "bf16": (at(out16),), "t24": (at(out32), self.t24_off, at(out24))}[kind]
            args = (self.a_ptr if a_ptr is None else a_ptr, c.lda, self.W_dev.data_ptr(), bias, c.K, c.width,
                    g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr()) + outs + (c.impl, ws.data_ptr(),
                                                                                             ws.numel(), _st())
        torch.cuda.synchronize()
        before = _lib.kernel_launches()
        _lib.call(entry, *args)
        torch.cuda.synchronize()
        raw = {"fp32": (out32,), "bf16": (out16,), "t24": (out32, out24)}[kind]
        return raw, _lib.kernel_launches() - before


def _within(got, ref, scale, tol, what):
    got = got.double().cpu()
    assert torch.isfinite(got).all(), "%s: non-finite values" % what
    if ref.numel() == 0:
        return 0.0
    ratio = ((got - ref).abs() / (tol * scale + 1e-30)).max().item()
    assert ratio <= 1.0, "%s: max |err| / bound = %.3g (tol %.1g)" % (what, ratio, tol)
    return ratio * tol


def _untouched(buf, keep, sentinel, what):
    """Every element of buf outside `keep` (a bool mask, or None: all) still holds the sentinel."""
    b = _bits(buf).cpu().to(torch.int64) & {1: 0xFF, 2: 0xFFFF, 4: 0xFFFFFFFF}[buf.element_size()]
    outside = b if keep is None else b[~keep]
    bad = (outside != sentinel).nonzero()
    assert bad.numel() == 0, "%s: %d elements outside the column blocks written (first at %s)" % (
        what, bad.numel(), bad[:4].flatten().tolist())


def check_case(name, kb_env=None):
    """Every entry point of one case against float64 (see the module docstring).  Returns ({entry: raw outputs},
    {entry: worst |err| / scale}, the Inputs)."""
    from tests.test_gpu_t24_tables import round_words
    inp = Inputs(name)
    c = inp.c
    outs, worst, fp32 = {}, {}, None
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for entry in entries(c):
        inst = case_instance(name, entry, kb_env)
        tag = "%s %s (%s P %s)" % (name, entry, inst.path, inst.P)
        raw, launches = inp.call(entry)
        assert launches == len(inst.launches), "%s: %d launches, restated %s" % (tag, launches, inst.launches)
        idx, ref, scale, lds = inp.reference(inst.P)
        tol = FWD_TOL[inst.P]
        n = inp.out_elems
        kind = out_kind(entry)
        outs[entry] = raw
        if kind == "fp32":
            buf = raw[0]
            keep = torch.zeros(n + 2 * HEAD, dtype=torch.bool)
            keep[HEAD + idx] = True
            _untouched(buf, keep, SENT32, tag)
            fp32 = buf[HEAD:HEAD + n].cpu()[idx]
            worst[entry] = _within(fp32, ref, scale, tol, tag)
        elif kind == "bf16":
            buf = raw[0]
            keep = torch.zeros(n + 2 * HEAD, dtype=torch.bool)
            keep[HEAD + idx] = True
            _untouched(buf, keep, SENT16, tag)
            got = buf[HEAD:HEAD + n].cpu()[idx]
            assert torch.equal(_bits(got), _bits(fp32.to(BF16))), "%s: not the RNE of the fp32 output" % tag
        else:
            b32, b24 = raw
            t0 = inp.t24_off
            f = idx < t0
            keep = torch.zeros(t0 + 2 * HEAD, dtype=torch.bool)
            keep[HEAD + idx[f]] = True
            _untouched(b32, keep, SENT32, tag + " fp32 blocks")
            assert torch.equal(_bits(b32[HEAD:HEAD + t0].cpu()[idx[f]]), _bits(fp32[f])), "%s: fp32 blocks" % tag
            hi, lo = _t24_bytes(idx[~f] - t0, lds[~f])
            keep = torch.zeros(b24.numel(), dtype=torch.bool)
            keep[HEAD + hi] = keep[HEAD + hi + 1] = keep[HEAD + lo] = True
            _untouched(b24, keep, SENT8, tag + " 24-bit planes")
            bytes_ = b24.cpu().to(torch.int64)
            words = (bytes_[HEAD + hi + 1] << 24) | (bytes_[HEAD + hi] << 16) | (bytes_[HEAD + lo] << 8)
            assert torch.equal(words, round_words(fp32[~f])), "%s: not the encoded fp32 output" % tag
            dec = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32).view(torch.float32)
            half_ulp = dec.double().abs() * 2.0 ** -16
            err = (dec.double() - ref[~f]).abs()
            assert (err <= tol * scale[~f] + half_ulp).all(), "%s: decoded 24-bit values out of bound" % tag
    # AF (fp32 A split in shared memory) equals the presplit kernel on k_split_bf16's halves of the same A
    main = entries(c)[0]
    if case_instance(name, main, kb_env).launches[-1][-1] is True:
        twin = case_instance(name, main, kb_env, a_off=c.a_off + 1)
        assert ("k_split_bf16", "A private") in twin.launches and twin.launches[-1][-1] is False
        a2 = torch.empty(inp.a_buf.numel() + 4, device=_dev())
        a2[1:1 + inp.a_buf.numel()] = inp.a_buf
        raw, launches = inp.call(main, a_ptr=a2.data_ptr() + (c.a_off + 1) * 4)
        assert launches == len(twin.launches), "%s split first: %d launches" % (name, launches)
        assert torch.equal(_bits(raw[0]), _bits(outs[main][0])), "%s: AF differs from the presplit kernel" % name
    print("\n%s (BN %d, %d SMs): worst |err| / scale %s" % (name, pick_tile_n(c.width), sms,
                                                             " ".join("%s %.2e" % kv for kv in worst.items())))
    return outs, worst, inp


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_linear_fwd_instance_matches_fp64(name):
    check_case(name, kb_env_of(os.environ.get("HGT_TC_P1_KB")))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the one-product k-blocks that only HGT_TC_P1_KB selects

def _p1_wide(name, kb):
    """Cases whose calls run the one-product kernel at 128 / 256 columns under HGT_TC_P1_KB=kb."""
    return any(k[0] == "k_typed_linear_tc" and k[1] != 64 and k[3] == 1
               for e in entries(CASES[name]) for k in case_instance(name, e, kb).launches)


@pytest.mark.gpu
@pytest.mark.parametrize("kb", [32, 64])
def test_p1_kblock_variant_matches_fp64_and_default(kb, tmp_path):
    """The one-product cases at 128 / 256 columns in a child process with HGT_TC_P1_KB=kb (the library reads it once per
    process): the same float64 checks there, and outputs bitwise equal to this process's (the other k-block, or the
    same one where kb is the default)."""
    assert kb_env_of(os.environ.get("HGT_TC_P1_KB")) is None
    names = [n for n in CASES if _p1_wide(n, kb)]
    assert len(names) >= 6
    path = tmp_path / "outputs.pt"
    env = dict(os.environ, HGT_TC_P1_KB=str(kb))
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_linear_fwd_instances", str(path)] + names, cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "child failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-6000:])
    assert ("child ok: %d cases" % len(names)) in r.stdout, r.stdout[-3000:]
    print(r.stdout)
    theirs = torch.load(path)
    for n in names:
        mine = check_case(n)[0]
        for entry, bufs in mine.items():
            for a, b in zip(bufs, theirs[n][entry]):
                assert torch.equal(_bits(a.cpu()), _bits(b)), "%s %s: KB %d differs from the default" % (n, entry, kb)


def _child(argv):
    path, names = argv[0], argv[1:]
    kb = kb_env_of(os.environ.get("HGT_TC_P1_KB"))
    res = {}
    for n in names:
        outs = check_case(n, kb)[0]
        res[n] = {e: tuple(t.cpu() for t in bufs) for e, bufs in outs.items()}
    torch.save(res, path)
    print("child ok: %d cases" % len(names))


if __name__ == "__main__":
    _child(sys.argv[1:])
