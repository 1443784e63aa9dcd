"""Every compiled instance of the small stages around the typed GEMMs against float64, at their edges.

Update epilogue (csrc/update.cu; hgt_update_epilogue, hgt_update_epilogue_dst and the pointer-table form inside
hgt_conv_forward): k_update_epilogue_vec<NV> (NV in {1, 2, 4, 8} float4 chunks per lane) when d % 4 == 0 and o, x, out,
norm_w, norm_b and bias are 16-byte aligned, the scalar k_update_epilogue otherwise.  `epilogue_instance` restates the
choice.
Update backward (csrc/update_bwd.cu): the atomic k_update_bwd<NPL> (NPL in {2, 4, 8, 16, 32} columns per lane), whose
128-row blocks (UB_WARPS * UB_ROWS_PER_WARP) sum d norm / d skip in shared memory when they hold one type and with
global atomics when they straddle types; the deterministic k_update_bwd_det<NPL> (512-row blocks inside one type) and
k_update_bwd_reduce.  `update_bwd_npl` and `update_bwd_block_kinds` restate the choices.
Weight fold (csrc/linear.cu): k_copy_linears (the W_q rows; hgt_concat_linears) and k_fold_pairs; its backward
(csrc/update_bwd.cu): k_fold_bwd_w + k_fold_bwd_rel (atomic), k_fold_bwd_w_det + k_fold_bwd_rel_det + k_fold_bwd_pri_det.
hgt_act_split (csrc/linear_bwd.cu): k_act_split with float4 or scalar loads, identity or exact-erf gelu, fp32 and / or
the bf16 hi / lo split.

test_case_lists_reach_every_instance (no GPU) checks that the case lists below reach every forward instance, both
backward kernels at every NPL and both block kinds.  Every GPU output starts as a sentinel (NaN for fp32, 7.0 for bf16,
or garbage where the header promises zero-initialisation), so an unwritten row and a write outside the addressed rows
both show.  The bf16 split is checked bitwise: hi = bf16_rne(out), lo = bf16_rne(out - hi), from the kernel's own fp32
output.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

# widths of the update epilogue and its backward: NV 1/2/4/8, lanes masked inside the last float4 chunk (32, 100, 132,
# 400, 1000), the scalar kernel for d % 4 != 0 (1, 3, 78), and NPL 2/4/8/16/32 in the backward
WIDTHS = [1, 3, 32, 64, 78, 100, 128, 132, 256, 400, 512, 1000, 1024]
# forward modes: "plain" (identity order, with the bf16 split where d % 8 == 0), "perm_active" (a row permutation with
# rows mapped to -1, and type_active), "dst" (hgt_update_epilogue_dst: type_dst + the a_linear bias), "misaligned"
# (o one float past a 16-byte boundary: the scalar kernel at any d, with perm and type_active)
EPILOGUE_MODES = ["plain", "perm_active", "dst", "misaligned"]

# rows per type of the forward cases: a type with 0 rows and a 1-row type; then rows of unknown type
FWD_COUNTS, FWD_UNKNOWN = [45, 0, 1, 20], 3
# backward: 128-row blocks 0-3 hold type 0 only, block 4 straddles types 0, 2 and 3, blocks 5 / 6 hold type 3 only and
# block 6 ends in unknown-type rows; type 0 spans two 512-row deterministic blocks
BWD_COUNTS, BWD_UNKNOWN = [600, 0, 1, 200], 7
UB_ROWS = 8 * 16          # UB_WARPS * UB_ROWS_PER_WARP, csrc/update_bwd.cu
UD_ROWS = 8 * 64          # UB_WARPS * UD_ROWS_PER_WARP

# weight fold shapes (d_in, d_out, H): d_k in {4, 8, 25, 26, 50, 64, 128, 256}, H = 1 and 32, d_in != d_out
FOLD_SHAPES = [(64, 128, 32), (40, 256, 32), (33, 100, 4), (50, 52, 2), (129, 400, 8), (129, 512, 8), (65, 128, 1),
               (48, 256, 1)]
# pairs (source type, relation) of the fold cases, T = 3, R = 3: two pairs each for types 0 and 2, none for type 1,
# none for relation 1
FOLD_T, FOLD_R = 3, 3
FOLD_PAIRS = [(0, 2), (2, 0), (0, 0), (2, 2)]

# hgt_act_split (rows, K, ld, offset of `in` in floats, what): ld > K and a misaligned `in` take the scalar loads
ACT_CASES = [(37, 64, 64, 0, "split"), (37, 256, 261, 0, "split"), (20, 8, 8, 1, "split"), (33, 128, 128, 1, "split"),
             (37, 30, 30, 0, "f32"), (19, 7, 9, 1, "f32")]


def epilogue_instance(d, aligned):
    """k_update_epilogue_vec<NV> as NV, or "scalar": csrc/update.cu hgt_update_epilogue_impl."""
    if not (aligned and d % 4 == 0 and d <= 1024):
        return "scalar"
    nv = (d // 4 + 31) // 32
    return next(v for v in (1, 2, 4, 8) if nv <= v)


def update_bwd_npl(d):
    """NPL of k_update_bwd / k_update_bwd_det: csrc/update_bwd.cu hgt_update_backward[_det]."""
    npl = (d + 31) // 32
    return next(v for v in (2, 4, 8, 16, 32) if npl <= v)


def _row0(counts, unknown):
    """type_row0 [T + 2]: prefix of the type counts, then the end of the unknown-type rows."""
    r = [0]
    for c in list(counts) + [unknown]:
        r.append(r[-1] + c)
    return r


def update_bwd_block_kinds(counts, unknown):
    """{"uniform", "mixed"} of k_update_bwd's 128-row blocks over known types."""
    row0 = _row0(counts, unknown)
    n, T = row0[-1], len(counts)

    def type_of(row):
        t = 0
        while t < T and row >= row0[t + 1]:
            t += 1
        return t

    kinds = set()
    for b0 in range(0, n, UB_ROWS):
        t0, t1 = type_of(b0), type_of(min(n, b0 + UB_ROWS) - 1)
        if t0 == t1 and t0 < T:
            kinds.add("uniform")
        elif t0 != t1:
            kinds.add("mixed")
    return kinds


def test_case_lists_reach_every_instance():
    """WIDTHS x EPILOGUE_MODES reach every epilogue instance, WIDTHS every backward NPL, BWD_COUNTS both block kinds
    and a type longer than one deterministic block, and ACT_CASES both load paths of k_act_split."""
    fwd = {epilogue_instance(d, mode != "misaligned") for d in WIDTHS for mode in EPILOGUE_MODES}
    assert fwd == {"scalar", 1, 2, 4, 8}
    assert {epilogue_instance(d, False) for d in WIDTHS if d % 4 == 0} == {"scalar"}
    assert {update_bwd_npl(d) for d in WIDTHS} == {2, 4, 8, 16, 32}
    assert update_bwd_block_kinds(BWD_COUNTS, BWD_UNKNOWN) == {"uniform", "mixed"}
    assert max(BWD_COUNTS) > UD_ROWS and 0 in BWD_COUNTS and 1 in BWD_COUNTS
    assert 0 in FWD_COUNTS and 1 in FWD_COUNTS and FWD_UNKNOWN > 0
    assert {dout // H for _, dout, H in FOLD_SHAPES} == {4, 8, 25, 26, 50, 64, 128, 256}
    assert {1, 32} <= {H for _, _, H in FOLD_SHAPES} and any(di != do for di, do, _ in FOLD_SHAPES)
    assert {t for t, _ in FOLD_PAIRS} == {0, 2} and {r for _, r in FOLD_PAIRS} == {0, 2}
    # float4 loads need a 16-byte aligned row start and 4 columns; the rest are scalar
    assert any(ld == K and off == 0 and K % 4 == 0 for _, K, ld, off, _ in ACT_CASES)
    assert any(ld % 4 or off for _, K, ld, off, _ in ACT_CASES)
    assert any(K % 4 for _, K, _, _, _ in ACT_CASES)


# ---------------------------------------------------------------------------------------------------------------------
def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from pyhgt_b200 import _lib as L
    return L


def _i32(v, dev):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def _nan(*shape, dev):
    return torch.full(shape, float("nan"), device=dev)


def _ptr_table(tensors, dev):
    """Device array of the tensors' device pointers (the per-type parameter tables the C ABI takes)."""
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64).to(dev)


def _rel_fro(got, ref, floor=1e-30):
    """|got - ref| / max(|ref|, floor) in the Frobenius norm.  floor: the scale of an output that is exactly zero in exact
    arithmetic (a LayerNorm over one column), where float64 leaves round-off and the kernel an exact zero."""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(floor))


def _scaled_max(got, ref, floor=1e-30):
    """max |got - ref| over max(max |ref|, floor): an elementwise error scaled to the output's magnitude."""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(floor)) if ref.numel() else 0.0


def _bf16_split(out):
    """The bf16 operand split of an fp32 tensor, round-to-nearest-even: (hi, lo) as int16 bit patterns."""
    hi = out.to(torch.bfloat16)
    lo = (out - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


# ---- update epilogue ------------------------------------------------------------------------------------------------
FWD_SKIP = [0.3, -0.7, -20.0, 20.0]      # type 3 saturates the gate: sigmoid(20) is 1.0 in fp32
N_BIG, N_CONST = 4, 2                    # LayerNorm edge rows at the start of type 3


def _epilogue_inputs(d, seed):
    """o, x [N, d] (CPU fp32), skip [T], norm_w / norm_b [T, d], a_linear bias [T, d].  The first rows of type 3 have
    mean 1e4 and std 1e-2 (they catch a one-pass E[y^2] - E[y]^2 variance), then constant rows (var 0); their x rows are
    0 and their gate is saturated, so y = o exactly in fp32 and in the float64 reference up to 2e-9."""
    gen = torch.Generator().manual_seed(seed)
    row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
    N, T = row0[-1], len(FWD_COUNTS)
    o, x = torch.randn(N, d, generator=gen), torch.randn(N, d, generator=gen)
    r3 = row0[3]
    o[r3:r3 + N_BIG] = 1e4 + 1e-2 * torch.randn(N_BIG, d, generator=gen)
    o[r3 + N_BIG:r3 + N_BIG + N_CONST] = 1.5
    x[r3:r3 + N_BIG + N_CONST] = 0.0
    skip = torch.tensor(FWD_SKIP)
    nw = 1.0 + 0.5 * torch.randn(T, d, generator=gen)
    nb = 0.5 * torch.randn(T, d, generator=gen)
    bias = torch.randn(T, d, generator=gen)
    return o, x, skip, nw, nb, bias


def _epilogue_ref(o, x, skip, nw, nb, type_dst, bias):
    """float64 update epilogue in rank order (conv.py:129-133); unknown-type rows are zeros."""
    row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
    T, d = len(FWD_COUNTS), o.shape[1]
    out = torch.zeros(o.shape, dtype=torch.float64)
    for t in range(T):
        r = slice(row0[t], row0[t + 1])
        ot = o[r].double().clone()
        if type_dst is not None:
            ot[type_dst[t]:] = bias[t].double()
        a = torch.sigmoid(skip[t].double()) if skip is not None else 1.0
        b = 1.0 - a if skip is not None else 1.0
        y = ot * a + x[r].double() * b
        if nw is not None:
            y = F.layer_norm(y, (d,), nw[t].double(), nb[t].double(), 1e-5)
        out[r] = y
    return out


def _epilogue_case(d, mode, seed):
    """The row layout of one forward mode: (perm list or None, type_active or None, type_dst or None, misaligned)."""
    row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
    N = row0[-1]
    perm = active = dst = None
    if mode in ("perm_active", "misaligned"):
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(seed + 7)).tolist()
        perm[row0[0] + 3] = -1                   # a known row and an unknown-type row without an output row
        perm[row0[4] + 1] = -1
        active = [30, 0, 1, 15]
    if mode == "dst":
        dst = [20, 0, 0, 12]                     # the 1-row type is all tail; the edge rows of type 3 are not
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(seed + 7)).tolist()
    return perm, active, dst, mode == "misaligned"


def _run_epilogue(o, x, skip, nw, nb, bias, perm, active, dst, misaligned, split, dev):
    """One hgt_update_epilogue[_dst] call: (out, hi, lo) with NaN / 7.0 sentinels in whatever it does not write."""
    L = _lib()
    N, d = o.shape
    T = len(FWD_COUNTS)
    o_d = o.clone()
    if dst is not None:                          # rows past type_dst[t]: `o` was never computed there
        row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
        for t in range(T):
            o_d[row0[t] + dst[t]:row0[t + 1]] = float("nan")
    if active is not None:                       # rows past type_active[t]: halo sources, `o` not computed
        row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
        for t in range(T):
            o_d[row0[t] + active[t]:row0[t + 1]] = float("nan")
    if misaligned:
        buf = torch.empty(N * d + 4, device=dev)
        o_dev = buf[1:1 + N * d].view(N, d)
        o_dev.copy_(o_d.to(dev))
    else:
        o_dev = o_d.to(dev)
    x_d, tr0 = x.to(dev), _i32(_row0(FWD_COUNTS, FWD_UNKNOWN), dev)
    out = _nan(N, d, dev=dev)
    hi = lo = None
    if split:
        hi = torch.full((N, d), 7.0, dtype=torch.bfloat16, device=dev)
        lo = torch.full((N, d), 7.0, dtype=torch.bfloat16, device=dev) if split == "pair" else None
    s_d = skip.to(dev) if skip is not None else None
    nw_d = nw.to(dev) if nw is not None else None
    nb_d = nb.to(dev) if nb is not None else None
    perm_d = _i32(perm, dev) if perm is not None else None
    ptr = L.ptr
    if dst is not None:
        dst_d, bias_d = _i32(dst, dev), bias.to(dev)     # named: a temporary's memory could be reused before the launch
        L.call("hgt_update_epilogue_dst", o_dev.data_ptr(), x_d.data_ptr(), tr0.data_ptr(), T, ptr(s_d), ptr(nw_d),
               ptr(nb_d), ptr(perm_d), dst_d.data_ptr(), bias_d.data_ptr(), N, d, out.data_ptr(), ptr(hi), ptr(lo),
               _st())
    else:
        act_d = _i32(active, dev) if active is not None else None
        L.call("hgt_update_epilogue", o_dev.data_ptr(), x_d.data_ptr(), tr0.data_ptr(), T, ptr(s_d), ptr(nw_d),
               ptr(nb_d), ptr(perm_d), ptr(act_d), N, d, out.data_ptr(), ptr(hi), ptr(lo), _st())
    torch.cuda.synchronize()
    return out.cpu(), (hi.cpu() if hi is not None else None), (lo.cpu() if lo is not None else None)


def _expected_rows(perm, active, N):
    """(rank row, output row) of every row the epilogue writes."""
    row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
    T = len(FWD_COUNTS)
    pairs = []
    for row in range(N):
        t = next((u for u in range(T) if row < row0[u + 1]), T)
        if active is not None and t < T and row - row0[t] >= active[t]:
            continue
        dst_row = row if perm is None else perm[row]
        if dst_row < 0:
            continue
        pairs.append((row, dst_row))
    return pairs


@pytest.mark.gpu
@pytest.mark.parametrize("mode", EPILOGUE_MODES)
@pytest.mark.parametrize("d", WIDTHS)
def test_update_epilogue_matches_fp64(d, mode):
    """Every row the epilogue addresses against float64, every other output row untouched, for skip on / off and
    LayerNorm on / off; with the bf16 split (d % 8 == 0, identity order) hi / lo bitwise, the hi-only call bitwise its
    hi half, and `out` bitwise the same with and without the split."""
    dev = _dev()
    o, x, skip, nw, nb, bias = _epilogue_inputs(d, seed=d)
    N = o.shape[0]
    perm, active, dst, misaligned = _epilogue_case(d, mode, seed=d)
    rows = _expected_rows(perm, active, N)
    src = torch.tensor([r for r, _ in rows])
    dst_rows = torch.tensor([w for _, w in rows])
    unwritten = torch.ones(N, dtype=torch.bool)
    unwritten[dst_rows] = False
    row0 = _row0(FWD_COUNTS, FWD_UNKNOWN)
    edge = torch.zeros(N, dtype=torch.bool)
    edge[row0[3]:row0[3] + N_BIG] = True                 # mean 1e4, std 1e-2: bounded on their own below
    split_ok = perm is None and active is None and d % 8 == 0
    for use_skip in (True, False):
        for use_norm in (True, False):
            s = skip if use_skip else None
            w, b = (nw, nb) if use_norm else (None, None)
            ref = _epilogue_ref(o, x, s, w, b, dst, bias)
            out, _, _ = _run_epilogue(o, x, s, w, b, bias, perm, active, dst, misaligned, None, dev)
            what = "d=%d %s skip=%s norm=%s" % (d, mode, use_skip, use_norm)
            assert torch.isnan(out[unwritten]).all(), what + ": a row outside the addressed rows was written"
            got, exp = out[dst_rows].double(), ref[src]
            big = edge[src] if use_norm else torch.zeros(len(src), dtype=torch.bool)
            # H100 (every width and mode): scaled max error <= 4.8e-7, relative Frobenius <= 1.5e-7
            e = (_scaled_max(got[~big], exp[~big]), _rel_fro(got[~big], exp[~big]))
            assert e[0] < 5e-6 and e[1] < 2e-6, (what, e)
            if big.any():
                # values of 1e4 are fp32 multiples of 2^-10 ~ 0.1 std, and so is the rounding of their mean: the
                # two-pass variance leaves scaled errors up to 0.115 on the H100 (d = 3; an fp32 emulation on the
                # CPU gives the same, up to 0.14), while E[y^2] - E[y]^2 gives NaN (a negative variance) or > 1
                e = _scaled_max(got[big], exp[big])
                assert e < 0.5, (what, "mean 1e4 / std 1e-2 rows", e)
            if split_ok:
                out_p, hi, lo = _run_epilogue(o, x, s, w, b, bias, perm, active, dst, misaligned, "pair", dev)
                out_h, hi_only, _ = _run_epilogue(o, x, s, w, b, bias, perm, active, dst, misaligned, "hi", dev)
                assert torch.equal(out_p.view(torch.int32), out.view(torch.int32)), what
                assert torch.equal(out_h.view(torch.int32), out.view(torch.int32)), what
                eh, el = _bf16_split(out)
                assert torch.equal(hi.view(torch.int16), eh), what + ": hi is not bf16_rne(out)"
                assert torch.equal(lo.view(torch.int16), el), what + ": lo is not bf16_rne(out - hi)"
                assert torch.equal(hi_only.view(torch.int16), eh), what + ": the hi-only split differs"


def _conv_and_graph(d, H, seed):
    from pyhgt_b200 import HGTConv, synth
    T, R = 3, 2
    g = synth.make_random(700, 4000, T, R, seed=seed, isolated_frac=0.3)
    torch.manual_seed(seed)
    conv = HGTConv(d, d, T, R, H, 0.2, True, True)
    with torch.no_grad():
        for n in conv.norms:                       # nn.LayerNorm starts at (1, 0): make the parameters matter
            n.weight.normal_(1.0, 0.3)
            n.bias.normal_(0.0, 0.3)
        conv.skip.normal_(0.0, 1.0)
    return conv, g, T, R


def _misalign_norms(conv, offset, dev):
    """Replace every norms[t].weight / .bias by a view at float offset `offset` (mod 4) into one flat buffer."""
    T, d = len(conv.norms), conv.out_dim
    flat = torch.zeros(offset + 2 * T * d + 4, device=dev)
    pos = offset
    for n in conv.norms:
        for name in ("weight", "bias"):
            p = getattr(n, name)
            view = flat[pos:pos + d]
            view.copy_(p.data)
            setattr(n, name, torch.nn.Parameter(view))
            pos += d
    return flat


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["offset1", "offset2", "offset3", "vector_to_parameters"])
@pytest.mark.parametrize("d,H", [(64, 4), (400, 8)])
def test_fused_forward_takes_misaligned_layernorm_parameters(d, H, layout):
    """The eval-mode fused forward (hgt_conv_forward) with LayerNorm parameters that are views at float offsets 1, 2, 3
    (mod 4) into a flat buffer, or after a parameters_to_vector -> vector_to_parameters round trip: against float64
    and against the per-stage path, which stacks the norms into a fresh tensor."""
    from oracle import hgt_oracle
    dev = _dev()
    conv, g, T, R = _conv_and_graph(d, H, seed=d + H)
    conv = conv.to(dev).eval()
    if layout == "vector_to_parameters":
        vec = torch.nn.utils.parameters_to_vector(conv.parameters())
        torch.nn.utils.vector_to_parameters(vec, conv.parameters())
    else:
        _misalign_norms(conv, int(layout[-1]), dev)
    assert all(n.weight.data_ptr() % 16 and n.bias.data_ptr() % 16 for n in conv.norms)
    x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(1))
    args = (x.to(dev), g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    with torch.no_grad():
        type(conv).fused_call = True
        try:
            fused = conv(*args)
            type(conv).fused_call = False
            staged = conv(*args)
        finally:
            type(conv).fused_call = True
    torch.cuda.synchronize()
    params = {k: v.detach().cpu() for k, v in conv.state_dict().items()}
    ref, _ = hgt_oracle.hgt_forward_dense_fp64(params, x, g.node_type, g.edge_index, g.edge_type, g.edge_time,
                                              num_types=T, num_relations=R, n_heads=H, use_norm=True, use_RTE=True)
    # H100: fused vs per-stage scaled max difference <= 2.0e-6; against float64 the 1e-3 of the parity suite
    e_staged, e_ref = _scaled_max(fused, staged), _scaled_max(fused, ref)
    assert e_staged < 2e-5, e_staged
    assert torch.allclose(fused.cpu().double(), ref, rtol=1e-3, atol=1e-3), e_ref


# ---- update backward ------------------------------------------------------------------------------------------------
BWD_ACTIVE = [450, 0, 1, 130]


def _update_bwd_inputs(d, seed):
    gen = torch.Generator().manual_seed(seed)
    row0 = _row0(BWD_COUNTS, BWD_UNKNOWN)
    N, T = row0[-1], len(BWD_COUNTS)
    o, x, g = (torch.randn(N, d, generator=gen) for _ in range(3))
    skip = torch.tensor([0.4, -1.0, 2.0, -0.3])
    nw = 1.0 + 0.5 * torch.randn(T, d, generator=gen)
    perm = torch.randperm(N, generator=gen).tolist()
    return o, x, g, skip, nw, perm


def _update_bwd_ref(o, x, g, skip, nw, perm, active):
    """float64 autograd of the epilogue with loss <out, g>: d o, d x, d skip, d norm_w, d norm_b."""
    row0 = _row0(BWD_COUNTS, BWD_UNKNOWN)
    T, d = len(BWD_COUNTS), o.shape[1]
    o64, x64 = o.double().requires_grad_(True), x.double().requires_grad_(True)
    s64 = (skip if skip is not None else torch.zeros(T)).double().requires_grad_(True)
    nw64 = (nw if nw is not None else torch.ones(T, d)).double().requires_grad_(True)
    nb64 = torch.zeros(T, d, dtype=torch.float64, requires_grad=True)
    pidx = torch.tensor(perm) if perm is not None else torch.arange(o.shape[0])
    g64 = g.double()[pidx]                           # dout is in original order: row `row` reads dout[perm[row]]
    loss = (s64.sum() + nw64.sum() + nb64.sum()) * 0
    for t in range(T):
        n_act = row0[t + 1] - row0[t] if active is None else active[t]
        r = slice(row0[t], row0[t] + n_act)
        a = torch.sigmoid(s64[t]) if skip is not None else 1.0
        b = 1.0 - a if skip is not None else 1.0
        y = o64[r] * a + x64[r] * b
        if nw is not None:
            y = F.layer_norm(y, (d,), nw64[t], nb64[t], 1e-5)
        loss = loss + (y * g64[r]).sum()
    loss.backward()
    return o64.grad, x64.grad, s64.grad, nw64.grad, nb64.grad


GARBAGE = 123.0


def _run_update_bwd(o, x, g, skip, nw, perm, active, det, dev, counts=BWD_COUNTS, unknown=BWD_UNKNOWN):
    """One hgt_update_backward[_det] call with NaN-filled d o / d x and garbage-filled d skip / d norm; for det the
    workspace is exactly the queried size, followed by guard bytes that must stay unchanged."""
    L = _lib()
    row0 = _row0(counts, unknown)
    N, T = row0[-1], len(counts)
    d = o.shape[1] if o.dim() == 2 else 1
    o_d = o.clone()
    if active is not None:                           # their `o` rows were never computed
        for t in range(T):
            o_d[row0[t] + active[t]:row0[t + 1]] = float("nan")
    o_d, x_d, g_d = o_d.to(dev), x.to(dev), g.to(dev)
    tr0 = _i32(row0, dev)
    # at least one row each, so that n_nodes == 0 still passes non-NULL buffers
    o_d, x_d, g_d = (t if N else torch.zeros(1, d, device=dev) for t in (o_d, x_d, g_d))
    d_o, d_x = _nan(max(N, 1), d, dev=dev), _nan(max(N, 1), d, dev=dev)
    d_s = torch.full((T,), GARBAGE, device=dev)
    d_nw, d_nb = torch.full((T, d), GARBAGE, device=dev), torch.full((T, d), GARBAGE, device=dev)
    s_d = skip.to(dev) if skip is not None else None
    nw_d = nw.to(dev) if nw is not None else None
    perm_d = _i32(perm, dev) if perm is not None else None
    act_d = _i32(active, dev) if active is not None else None
    ptr = L.ptr
    common = (g_d.data_ptr(), o_d.data_ptr(), x_d.data_ptr(), tr0.data_ptr(), T, ptr(s_d), ptr(nw_d), ptr(perm_d),
              ptr(act_d), N, d, d_o.data_ptr(), d_x.data_ptr(), d_s.data_ptr(),
              d_nw.data_ptr() if nw is not None else None, d_nb.data_ptr() if nw is not None else None)
    guard_ok = True
    if det:
        need = ctypes.c_size_t()
        L.call("hgt_update_backward_det_workspace_bytes", N, T, d, ctypes.byref(need))
        buf = torch.full((need.value + 256,), 0xA5, dtype=torch.uint8, device=dev)
        L.call("hgt_update_backward_det", *common, buf.data_ptr(), need.value, _st())
        torch.cuda.synchronize()
        guard_ok = bool((buf[need.value:] == 0xA5).all())
    else:
        L.call("hgt_update_backward", *common, _st())
    torch.cuda.synchronize()
    return d_o[:N].cpu(), d_x[:N].cpu(), d_s.cpu(), d_nw.cpu(), d_nb.cpu(), guard_ok


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d", WIDTHS)
def test_update_backward_matches_fp64(d, det):
    """d o, d x, d skip, d norm_w, d norm_b of the atomic and the deterministic update backward against float64
    autograd, with skip, LayerNorm, perm and type_active each on and off.  Rows past type_active and unknown-type rows
    get exact zeros; d skip is untouched without skip; the det path repeats bitwise and stays inside its workspace."""
    dev = _dev()
    o, x, g, skip, nw, perm_all = _update_bwd_inputs(d, seed=3 * d + det)
    row0 = _row0(BWD_COUNTS, BWD_UNKNOWN)
    T = len(BWD_COUNTS)
    for use_skip in (True, False):
        for use_norm in (True, False):
            for sharded in (False, True):
                s = skip if use_skip else None
                w = nw if use_norm else None
                perm = perm_all if sharded else None
                active = BWD_ACTIVE if sharded else None
                what = "d=%d det=%s skip=%s norm=%s perm/active=%s" % (d, det, use_skip, use_norm, sharded)
                got = _run_update_bwd(o, x, g, s, w, perm, active, det, dev)
                ref = _update_bwd_ref(o, x, g, s, w, perm, active)
                d_o, d_x, d_s, d_nw, d_nb, guard_ok = got
                assert guard_ok, what + ": the det backward wrote past its workspace"
                zero = torch.zeros(row0[-1], dtype=torch.bool)
                zero[row0[T]:] = True
                if active is not None:
                    for t in range(T):
                        zero[row0[t] + active[t]:row0[t + 1]] = True
                assert (d_o[zero] == 0).all() and (d_x[zero] == 0).all(), what + ": rows without output not zero"
                # the gradients are O(1) or exactly zero (d = 1 under LayerNorm): errors are scaled to at least 1
                # H100: scaled max error <= 1.5e-5 (d o, d = 3) / 7.9e-6 (d x), relative Frobenius <= 1.0e-5
                for name, a, r in (("d_o", d_o, ref[0]), ("d_x", d_x, ref[1])):
                    assert not torch.isnan(a).any(), what + ": %s has unwritten rows" % name
                    e = (_scaled_max(a, r, 1.0), _rel_fro(a, r, 1.0))
                    assert e[0] < 1.5e-4 and e[1] < 1e-4, (what, name, e)
                if use_skip:
                    # a sum over all rows of a type: bounded relative to the vector's norm.  H100: <= 1.4e-5
                    e = _rel_fro(d_s, ref[2], 1.0)
                    assert e < 1.5e-4, (what, "d_skip", e)
                    assert d_s[1] == 0, what + ": the empty type's d_skip"
                else:
                    assert (d_s == GARBAGE).all(), what + ": d_skip touched in residual mode"
                if use_norm:
                    for name, a, r in (("d_norm_w", d_nw, ref[3]), ("d_norm_b", d_nb, ref[4])):
                        # H100: scaled max error <= 4.5e-7, relative Frobenius <= 4.3e-7
                        e = (_scaled_max(a, r, 1.0), _rel_fro(a, r, 1.0))
                        assert e[0] < 5e-6 and e[1] < 5e-6, (what, name, e)
                        assert (a[1] == 0).all(), what + ": the empty type's " + name
                if det and use_skip and use_norm:
                    again = _run_update_bwd(o, x, g, s, w, perm, active, det, dev)
                    for a, b in zip(got[:5], again[:5]):
                        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what + ": not bitwise repeatable"


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
def test_update_backward_zero_rows_zero_initialises(det):
    """With n_nodes == 0 the d skip / d norm outputs are still zero-initialised, as the header promises."""
    dev = _dev()
    d, T = 64, 4
    empty = torch.zeros(0, d)
    got = _run_update_bwd(empty, empty, empty, torch.ones(T), torch.ones(T, d), None, None, det, dev,
                          counts=[0] * T, unknown=0)
    assert (got[2] == 0).all() and (got[3] == 0).all() and (got[4] == 0).all() and got[5]


# ---- weight fold ----------------------------------------------------------------------------------------------------
def _fold_layout(d_out):
    """W_cat row starts of the W_q blocks (q_row0 [T]) and the pairs' K'/V' blocks (cat_row0 [P]), neither in ascending
    order, with 3 uncovered rows after every block; and the total row count."""
    order = [("p", 2), ("q", 1), ("p", 0), ("q", 2), ("p", 3), ("q", 0), ("p", 1)]
    q_row0, cat_row0 = [0] * FOLD_T, [0] * len(FOLD_PAIRS)
    pos = 0
    for kind, k in order:
        if kind == "q":
            q_row0[k] = pos
            pos += d_out + 3
        else:
            cat_row0[k] = pos
            pos += 2 * d_out + 3
    assert q_row0 != sorted(q_row0) or cat_row0 != sorted(cat_row0)
    return q_row0, cat_row0, pos


def _fold_params(d_in, d_out, H, seed):
    gen = torch.Generator().manual_seed(seed)
    dk = d_out // H
    T, R = FOLD_T, FOLD_R
    p = {n: torch.randn(T, d_out, d_in, generator=gen) / math.sqrt(d_in) for n in ("wq", "wk", "wv")}
    p.update({n: torch.randn(T, d_out, generator=gen) for n in ("bq", "bk", "bv")})
    p["att"] = torch.randn(R, H, dk, dk, generator=gen) / math.sqrt(dk)
    p["msg"] = torch.randn(R, H, dk, dk, generator=gen) / math.sqrt(dk)
    p["pri"] = 1.0 + 0.5 * torch.randn(R, H, generator=gen)
    return p


def _fold_ref(p, H):
    """float64 K'_p / V'_p weights and biases of every pair (include/hgt_b200.h, hgt_fold_weights):
    K'[h*dk+c, :] = pri[r,h] / sqrt(dk) * sum_a att[r,h,a,c] W_k[h*dk+a, :]; V' the same with msg and no scale."""
    T, d_out, d_in = p["wk"].shape
    dk = d_out // H
    out = []
    for t, r in FOLD_PAIRS:
        s = (p["pri"][r] / math.sqrt(dk))[:, None, None]
        wk = p["wk"][t].view(H, dk, d_in)
        wv = p["wv"][t].view(H, dk, d_in)
        kw = (torch.einsum("hac,had->hcd", p["att"][r], wk) * s).reshape(d_out, d_in)
        kb = (torch.einsum("hac,ha->hc", p["att"][r], p["bk"][t].view(H, dk)) * s[:, :, 0]).reshape(d_out)
        vw = torch.einsum("hac,had->hcd", p["msg"][r], wv).reshape(d_out, d_in)
        vb = torch.einsum("hac,ha->hc", p["msg"][r], p["bv"][t].view(H, dk)).reshape(d_out)
        out.append((kw, kb, vw, vb))
    return out


def _fold_dev(p, dev):
    """Per-type parameter tensors on the device and their pointer tables."""
    per = {n: [p[n][t].contiguous().to(dev) for t in range(FOLD_T)] for n in ("wq", "bq", "wk", "bk", "wv", "bv")}
    tabs = {n: _ptr_table(v, dev) for n, v in per.items()}
    return per, tabs


@pytest.mark.gpu
@pytest.mark.parametrize("d_in,d_out,H", FOLD_SHAPES)
def test_fold_weights_matches_fp64(d_in, d_out, H):
    """hgt_fold_weights: W_q rows bitwise copies, K'/V' rows against the float64 formula, uncovered W_cat rows keep
    their NaN sentinel; hgt_concat_linears bitwise."""
    dev = _dev()
    L = _lib()
    p = _fold_params(d_in, d_out, H, seed=d_in + d_out + H)
    q_row0, cat_row0, rows = _fold_layout(d_out)
    per, tabs = _fold_dev(p, dev)
    w_cat, b_cat = _nan(rows, d_in, dev=dev), _nan(rows, dev=dev)
    pt, pr = _i32([t for t, _ in FOLD_PAIRS], dev), _i32([r for _, r in FOLD_PAIRS], dev)
    rel = [p[n].to(dev) for n in ("att", "msg", "pri")]
    c0, q0 = _i32(cat_row0, dev), _i32(q_row0, dev)
    L.call("hgt_fold_weights", tabs["wq"].data_ptr(), tabs["bq"].data_ptr(), tabs["wk"].data_ptr(),
           tabs["bk"].data_ptr(), tabs["wv"].data_ptr(), tabs["bv"].data_ptr(), rel[0].data_ptr(), rel[1].data_ptr(),
           rel[2].data_ptr(), FOLD_T, FOLD_R, H, d_in, d_out, len(FOLD_PAIRS), pt.data_ptr(), pr.data_ptr(),
           c0.data_ptr(), q0.data_ptr(), w_cat.data_ptr(), b_cat.data_ptr(), _st())
    torch.cuda.synchronize()
    w_cat, b_cat = w_cat.cpu(), b_cat.cpu()
    covered = torch.zeros(rows, dtype=torch.bool)
    for t in range(FOLD_T):
        r = slice(q_row0[t], q_row0[t] + d_out)
        covered[r] = True
        assert torch.equal(w_cat[r].view(torch.int32), p["wq"][t].view(torch.int32))
        assert torch.equal(b_cat[r].view(torch.int32), p["bq"][t].view(torch.int32))
    p64 = {k: v.double() for k, v in p.items()}
    for i, (kw, kb, vw, vb) in enumerate(_fold_ref(p64, H)):
        k0, v0 = cat_row0[i], cat_row0[i] + d_out
        covered[k0:v0 + d_out] = True
        for name, got, ref in (("K'", w_cat[k0:v0], kw), ("K' bias", b_cat[k0:v0], kb),
                               ("V'", w_cat[v0:v0 + d_out], vw), ("V' bias", b_cat[v0:v0 + d_out], vb)):
            # H100: scaled max error <= 7.4e-7, relative Frobenius <= 3.0e-7
            e = (_scaled_max(got, ref), _rel_fro(got, ref))
            assert e[0] < 8e-6 and e[1] < 3e-6, (i, name, e)
    assert torch.isnan(w_cat[~covered]).all() and torch.isnan(b_cat[~covered]).all()
    assert not torch.isnan(w_cat[covered]).any()

    w2, b2 = _nan(FOLD_T * d_out + 5, d_in, dev=dev), _nan(FOLD_T * d_out + 5, dev=dev)
    L.call("hgt_concat_linears", tabs["wk"].data_ptr(), tabs["bk"].data_ptr(), FOLD_T, d_out, d_in, w2.data_ptr(),
           b2.data_ptr(), _st())
    torch.cuda.synchronize()
    n = FOLD_T * d_out
    assert torch.equal(w2[:n].cpu().view(torch.int32), p["wk"].reshape(n, d_in).view(torch.int32))
    assert torch.equal(b2[:n].cpu().view(torch.int32), p["bk"].reshape(n).view(torch.int32))
    assert torch.isnan(w2[n:]).all() and torch.isnan(b2[n:]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d_in,d_out,H", FOLD_SHAPES)
def test_fold_backward_matches_fp64(d_in, d_out, H, det):
    """hgt_fold_backward[_det] against float64 autograd of the fold with loss <W_cat, G> + <b_cat, g> over the K'/V'
    rows.  G is NaN on the W_q and uncovered rows (never read), all seven outputs start as garbage, and the type and
    relation without a pair come out exactly zero."""
    dev = _dev()
    L = _lib()
    p = _fold_params(d_in, d_out, H, seed=d_in + 2 * d_out + H)
    q_row0, cat_row0, rows = _fold_layout(d_out)
    gen = torch.Generator().manual_seed(d_out)
    G = torch.full((rows, d_in), float("nan"))
    gb = torch.full((rows,), float("nan"))
    for c0 in cat_row0:
        G[c0:c0 + 2 * d_out] = torch.randn(2 * d_out, d_in, generator=gen)
        gb[c0:c0 + 2 * d_out] = torch.randn(2 * d_out, generator=gen)
    p64 = {k: v.double().requires_grad_(True) for k, v in p.items()}
    loss = 0
    for i, (kw, kb, vw, vb) in enumerate(_fold_ref(p64, H)):
        k0, v0 = cat_row0[i], cat_row0[i] + d_out
        loss = loss + (kw * G[k0:v0].double()).sum() + (kb * gb[k0:v0].double()).sum()
        loss = loss + (vw * G[v0:v0 + d_out].double()).sum() + (vb * gb[v0:v0 + d_out].double()).sum()
    loss.backward()
    per, tabs = _fold_dev(p, dev)
    rel = [p[n].to(dev) for n in ("att", "msg", "pri")]
    pt, pr, c0 = (_i32([t for t, _ in FOLD_PAIRS], dev), _i32([r for _, r in FOLD_PAIRS], dev), _i32(cat_row0, dev))
    G_d, gb_d = G.to(dev), gb.to(dev)
    dk = d_out // H

    def run():
        outs = [torch.full(s, GARBAGE, device=dev) for s in
                ((FOLD_T, d_out, d_in), (FOLD_T, d_out), (FOLD_T, d_out, d_in), (FOLD_T, d_out),
                 (FOLD_R, H, dk, dk), (FOLD_R, H, dk, dk), (FOLD_R, H))]
        L.call("hgt_fold_backward_det" if det else "hgt_fold_backward", G_d.data_ptr(), gb_d.data_ptr(),
               tabs["wk"].data_ptr(), tabs["bk"].data_ptr(), tabs["wv"].data_ptr(), tabs["bv"].data_ptr(),
               rel[0].data_ptr(), rel[1].data_ptr(), rel[2].data_ptr(), FOLD_T, FOLD_R, H, d_in, d_out,
               len(FOLD_PAIRS), pt.data_ptr(), pr.data_ptr(), c0.data_ptr(), *[o.data_ptr() for o in outs], _st())
        torch.cuda.synchronize()
        return [o.cpu() for o in outs]

    got = run()
    names = ["d_wk", "d_bk", "d_wv", "d_bv", "d_att", "d_msg", "d_pri"]
    refs = [p64[n].grad for n in ("wk", "bk", "wv", "bv", "att", "msg", "pri")]
    for name, a, r in zip(names, got, refs):
        assert not torch.isnan(a).any(), name
        # H100: relative Frobenius <= 3.1e-7, scaled max error <= 5.2e-7; d_pri, a long mixed-sign sum, is bounded
        # relative to its norm only (as FRO_BOUND does): <= 2.1e-6
        e = _rel_fro(a, r)
        assert e < (2e-5 if name == "d_pri" else 3e-6), (name, e)
        if name != "d_pri":
            e = _scaled_max(a, r)
            assert e < 5e-6, (name, e)
    for a in got[:4]:
        assert (a[1] == 0).all(), "the type without a pair"
    for a in got[4:]:
        assert (a[1] == 0).all(), "the relation without a pair"
    if det:
        again = run()
        for a, b in zip(got, again):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- hgt_act_split --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("rows,K,ld,off,what", ACT_CASES)
def test_act_split_matches_fp64(rows, K, ld, off, what, act):
    """hgt_act_split: act(in) against float64 (exact-erf gelu for act 1), the bf16 hi / lo split bitwise from the
    fp32 output, the hi-only split bitwise its hi half, and nothing written past the [rows, K] outputs."""
    dev = _dev()
    L = _lib()
    gen = torch.Generator().manual_seed(rows * K + ld + off)
    src = 3.0 * torch.randn(rows, ld, generator=gen)
    buf = torch.empty(off + rows * ld + 4, device=dev)
    a_in = buf[off:off + rows * ld].view(rows, ld)
    a_in.copy_(src.to(dev))
    pad = 16
    out = _nan(rows * K + pad, dev=dev)
    ref = src[:, :K].double()
    if act:
        ref = F.gelu(ref)

    def bf(n):
        return torch.full((n,), 7.0, dtype=torch.bfloat16, device=dev)

    hi = lo = None
    if what == "split":
        hi, lo = bf(rows * K + pad), bf(rows * K + pad)
    L.call("hgt_act_split", a_in.data_ptr(), ld, rows, K, act, out.data_ptr(), L.ptr(hi), L.ptr(lo), _st())
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.isnan(out[rows * K:]).all()
    got = out[:rows * K].view(rows, K)
    # H100: scaled max error <= 4.6e-8, relative Frobenius <= 3.5e-8
    e = (_scaled_max(got, ref), _rel_fro(got, ref))
    assert e[0] < 5e-7 and e[1] < 4e-7, e
    if what == "split":
        hi, lo = hi.cpu(), lo.cpu()
        eh, el = _bf16_split(got.reshape(-1))
        assert torch.equal(hi[:rows * K].view(torch.int16), eh), "hi is not bf16_rne(act(in))"
        assert torch.equal(lo[:rows * K].view(torch.int16), el), "lo is not bf16_rne(act(in) - hi)"
        assert (hi[rows * K:] == 7.0).all() and (lo[rows * K:] == 7.0).all()
        hi_only = bf(rows * K + pad)
        L.call("hgt_act_split", a_in.data_ptr(), ld, rows, K, act, None, hi_only.data_ptr(), None, _st())
        torch.cuda.synchronize()
        assert torch.equal(hi_only.cpu().view(torch.int16), hi.view(torch.int16)), "the hi-only split differs"
