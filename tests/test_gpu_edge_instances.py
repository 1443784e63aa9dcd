"""Every compiled instance of the fused edge kernels against float64 on the same tables, widened.

The edge forward (csrc/edge.cu) and backward (csrc/edge_bwd.cu) are compiled once per lane map <VEC, NCH> (VEC in
{1, 2, 4} floats per load, NCH in {1, 2, 4, 8} chunks per lane), per table element type (fp32 tables through
hgt_edge_forward / hgt_edge_backward, bf16 tables through the _bf16 entry points), per forward data path (variant 1:
register gather k_edge_fwd_ldg; variant 2: the TMA ring k_edge_fwd_tma, which falls back to variant 1 when fewer than two
ring stages fit or a [K'|V'] row is not a multiple of 16 bytes) and per backward path (atomic k_edge_bwd; deterministic
k_edge_bwd_dst + k_edge_bwd_rows).  The instance is chosen from (d, H) alone; `lane_map` and `ring_fallback` below
restate that choice, and test_shape_list_reaches_every_instance (no GPU needed) checks that SHAPES reaches all 12 lane
maps and both ring fallbacks for both table types.

Every graph has a hub destination above plan.TILE_SPLIT_EDGES, so the split-destination path (k_merge_partials in the
forward, atomic dq or the piece merge in the backward) runs at every instance.  Each shape runs with RTE off and on.  The
"hot" cases scale Q so that the scores of one destination spread over far more than 100: most exp terms underflow in
fp32, which exercises the online rescale, the hub pieces' log-sum-exp merge and the backward's use of the saved (m, l).
"""
import ctypes
import math

import pytest
import torch

from pyhgt_b200 import _lib, plan as P, synth

# (d, H) with the lane map <VEC, NCH> each reaches (d_k = d / H)
SHAPES = [
    (16, 4), (32, 8),                 # <1,1>: d_k 4
    (40, 8),                          # <1,2>: d_k 5
    (100, 4), (75, 3),                # <1,4>: d_k 25; d = 75 rows are not 16-byte multiples (variant 2 -> 1)
    (200, 8),                         # <1,8>: d_k 25, chunk 7 masked
    (64, 4),                          # <2,1>: d_k 16
    (100, 2),                         # <2,2>: d_k 50
    (208, 8),                         # <2,4>: d_k 26
    (250, 5), (400, 8),               # <2,8>: d_k 50, odd head count / 8 heads
    (96, 3), (128, 8),                # <4,1>: a 4th head's lanes idle / 8 heads
    (256, 8), (256, 1), (256, 32),    # <4,2>: LPH 4, 32 and 1
    (512, 8),                         # <4,4>: d_k 64 (the ogbn-mag recipe); fp32 with RTE: fewer than 2 ring stages
    (1024, 8),                        # <4,8>: d_k 128, variant 1 with EDGE_UNROLL 1; fp32: fewer than 2 ring stages
]
# one shape per lane map for the hot-score cases
HOT_SHAPES = [(32, 8), (40, 8), (100, 4), (200, 8), (64, 4), (100, 2), (208, 8), (400, 8), (128, 8), (256, 8),
              (512, 8), (1024, 8)]
CASES = [(d, H, rte, False) for d, H in SHAPES for rte in (False, True)] + [(d, H, True, True) for d, H in HOT_SHAPES]
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def lane_map(d, H):
    """<VEC, NCH> of the edge kernels for (d, H): csrc/edge.cu:719-739 (forward) and csrc/edge_bwd.cu:439-455
    (lane_map, every backward pass)."""
    dk = d // H
    hp = 1
    while hp < H:
        hp <<= 1
    lph = 32 // hp
    vec = next((v for v in (4, 2) if dk % v == 0 and dk // v >= lph), 1)
    chunks = -(-dk // (vec * lph))
    nch = 1
    while nch < chunks:
        nch <<= 1
    return vec, nch


def ring_fallback(d, H, rte, kv_bytes):
    """Why a variant-2 forward runs variant 1 instead ("stages": fewer than 2 ring stages fit, "align": a [K'|V'] row is
    not a multiple of 16 bytes), or None: csrc/edge.cu:744-754 (kWarpsPerCta = 16, edge.cu:27)."""
    vec, nch = lane_map(d, H)
    row = 2 * d * kv_bytes
    slot = 2 * row if rte else row
    budget = 100 * 1024 if vec * nch <= 4 else 200 * 1024
    if min(budget // (16 * slot), 8) < 2:
        return "stages"
    return "align" if row % 16 else None


def test_shape_list_reaches_every_instance():
    """SHAPES reaches every <VEC, NCH> instance and both ring fallbacks for both table types, and HOT_SHAPES has one
    shape per instance."""
    every = {(v, n) for v in (1, 2, 4) for n in (1, 2, 4, 8)}
    assert {lane_map(d, H) for d, H in SHAPES} == every
    assert sorted(lane_map(d, H) for d, H in HOT_SHAPES) == sorted(every)
    for kv_bytes in (4, 2):
        reasons = {ring_fallback(d, H, rte, kv_bytes) for d, H, rte, _ in CASES}
        assert {"stages", "align", None} <= reasons, (kv_bytes, reasons)
    assert ring_fallback(512, 8, True, 4) == "stages"       # the ogbn-mag layer, fp32
    assert ring_fallback(1024, 8, True, 2) == "stages"


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _graph(T, R, n_nodes=900, n_edges=6000, hub_edges=2500, seed=0):
    """Random typed graph with one hub destination above the split threshold."""
    g = synth.make_random(n_nodes, n_edges, T, R, seed=seed, self_loops=20)
    gen = torch.Generator().manual_seed(seed + 1)
    hub = 3
    src = torch.cat([g.edge_index[0], torch.randint(0, n_nodes, (hub_edges,), generator=gen)])
    dst = torch.cat([g.edge_index[1], torch.full((hub_edges,), hub, dtype=torch.int64)])
    g.edge_index = torch.stack([src, dst])
    g.edge_type = torch.cat([g.edge_type, torch.randint(0, R, (hub_edges,), generator=gen)])
    g.edge_time = torch.cat([g.edge_time, torch.randint(0, 240, (hub_edges,), generator=gen)])
    assert hub_edges > P.TILE_SPLIT_EDGES
    return g


def _plan(d, H, rte, seed):
    dev = _dev()
    T, R = 3, 2
    g = _graph(T, R, seed=seed)
    plan = P.build_plan(g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev),
                        g.edge_time.to(dev) if rte else None, T, R)
    assert plan.n_split > 0
    return plan, T


def _q_scale(d, H, hot):
    """1, or for the hot cases a Q scale that gives scores of standard deviation ~60: the scores of one destination then
    spread over several hundred, and exp(s - max) underflows to 0 in fp32 for most terms."""
    return 60.0 / math.sqrt(d // H) if hot else 1.0


def _tables(plan, d, rte, seed, dtype, q_scale=1.0):
    """Q fp32 [N, d] and [K'|V'] / RTE tables of `dtype` with their trailing all-zero row."""
    dev = _dev()
    gen = torch.Generator().manual_seed(seed)
    q = (q_scale * torch.randn(plan.n_nodes, d, generator=gen)).to(dev)
    kv = torch.randn(plan.kv_rows + 1, 2 * d, generator=gen).to(dtype).to(dev)
    kv[-1].zero_()
    kvr = None
    if rte:
        kvr = (0.5 * torch.randn(plan.n_pairs * P.RTE_MAX_LEN + 1, 2 * d, generator=gen)).to(dtype).to(dev)
        kvr[-1].zero_()
    return q, kv, kvr


def _edge_ref(plan, q, kv, kvr, H):
    """float64 edge attention on the given (widened) tables: agg [N, d], att per CSR position [E, H], (m, l) [N, H]."""
    N, d = q.shape
    dk = d // H
    rp = plan.row_ptr.cpu().long()
    E = int(rp[-1])
    dst = torch.repeat_interleave(torch.arange(N), rp[1:] - rp[:-1])
    kr = plan.kv_row[:E].cpu().long()
    kk, vv = kv[kr, :d], kv[kr, d:]
    if kvr is not None:
        rr = plan.rte_row[:E].cpu().long()
        kk, vv = kk + kvr[rr, :d], vv + kvr[rr, d:]
    s = (q[dst].view(E, H, dk) * kk.view(E, H, dk)).sum(-1)
    m = torch.full((N, H), -float("inf"), dtype=s.dtype).index_reduce_(0, dst, s.detach(), "amax")
    p = torch.exp(s - m[dst])
    l = torch.zeros(N, H, dtype=s.dtype).index_add(0, dst, p)
    att = p / (l[dst] + 1e-16)
    agg = torch.zeros(N, H, dk, dtype=s.dtype).index_add(0, dst, att[:, :, None] * vv.view(E, H, dk)).view(N, d)
    return agg, att, m, l


def _forward(plan, T, q, kv, kvr, d, H, variant, att=None, dtype="fp32"):
    """hgt_edge_forward[_bf16]: agg, stats [N, 2H] (and att when given)."""
    dev = _dev()
    N, E = plan.n_nodes, plan.n_edges
    agg = torch.full((N, d), float("nan"), device=dev)
    stats = torch.empty(N, 2 * H, device=dev)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    rte = kvr is not None
    _lib.call("hgt_edge_forward" + ("_bf16" if dtype == "bf16" else ""), q.data_ptr(), kv.data_ptr(),
              _lib.ptr(kvr), plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
              plan.rte_row.data_ptr() if rte else None, plan.csr_eid.data_ptr(), plan.tiles.data_ptr(), plan.n_tiles,
              plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, N, E, d, H, 0, agg.data_ptr(), _lib.ptr(att),
              stats.data_ptr(), None, None, ws.data_ptr(), ws.numel(), variant, _lib.ptr(plan.tile_counts_dev),
              plan.type_row0_dev.data_ptr(), T, None, _st())
    return agg, stats


def _check_hot(att_ref):
    """The hot cases really are in the underflow regime: most normalised weights lie below fp32's exp range."""
    frac = float((att_ref < math.exp(-88.0)).double().mean())
    assert frac > 0.5, "only %.2f of the attention weights underflow" % frac


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("d,H,rte,hot", CASES)
def test_edge_forward_matches_fp64(d, H, rte, hot, variant, dtype):
    """agg, att and the saved (m, l) of one edge forward against float64 on the same tables."""
    plan, T = _plan(d, H, rte, seed=d + H)
    q, kv, kvr = _tables(plan, d, rte, d, DTYPES[dtype], _q_scale(d, H, hot))
    N, E = plan.n_nodes, plan.n_edges
    att = torch.empty(E, H, device=q.device)
    agg, stats = _forward(plan, T, q, kv, kvr, d, H, variant, att, dtype)
    torch.cuda.synchronize()
    ref, att_ref, m_ref, l_ref = _edge_ref(plan, q.cpu().double(), kv.cpu().double(),
                                           None if kvr is None else kvr.cpu().double(), H)
    if hot:
        _check_hot(att_ref)
    has_in = (plan.row_ptr[1:] - plan.row_ptr[:-1]).cpu() > 0
    # hot: the fp32 rounding error of a score grows with its size (~60 instead of ~1); on an H100 it moved m by up to
    # 2.4e-5 and, through near-tied softmax weights, agg by up to 3.9e-5
    atol = 1e-4 if hot else 1e-5
    torch.testing.assert_close(agg.cpu().double(), ref, rtol=1e-4, atol=atol)
    eid = plan.csr_eid[:E].cpu().long()
    torch.testing.assert_close(att.cpu().double()[eid], att_ref, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(stats[:, :H].cpu().double()[has_in], m_ref[has_in], rtol=1e-5, atol=atol)
    torch.testing.assert_close(stats[:, H:].cpu().double()[has_in], l_ref[has_in], rtol=1e-4, atol=1e-5)


def _max_err(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("d,H,rte,hot", CASES)
def test_edge_backward_matches_fp64(d, H, rte, hot, det, dtype):
    """dq, d[K'|V'] and d RTE of the atomic and the deterministic edge backward against float64 autograd; the
    deterministic path repeats bitwise."""
    from pyhgt_b200.autograd import _edge_backward_det
    dev = _dev()
    plan, T = _plan(d, H, rte, seed=2 * d + H)
    q, kv, kvr = _tables(plan, d, rte, d + 1, DTYPES[dtype], _q_scale(d, H, hot))
    N = plan.n_nodes
    agg, stats = _forward(plan, T, q, kv, kvr, d, H, 0, None, dtype)
    dagg = torch.randn(N, d, generator=torch.Generator().manual_seed(5)).to(dev)
    sfx = "_bf16" if dtype == "bf16" else ""

    def run():
        dq = torch.empty(N, d, device=dev)
        dkv = torch.empty(plan.kv_rows + 1, 2 * d, device=dev)
        dkvr = torch.empty_like(kvr, dtype=torch.float32) if rte else None
        if det:
            _edge_backward_det(q, kv, kvr, agg, dagg, stats, plan, d, H, dq, dkv, dkvr, sfx)
        else:
            w2 = torch.empty(256, dtype=torch.uint8, device=dev)
            _lib.call("hgt_edge_backward" + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(),
                      dagg.data_ptr(), stats.data_ptr(), plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
                      plan.rte_row.data_ptr() if rte else None, plan.tiles.data_ptr(), plan.n_tiles, N, d, H,
                      plan.kv_rows + 1, kvr.shape[0] if rte else 0, dq.data_ptr(), dkv.data_ptr(), _lib.ptr(dkvr),
                      w2.data_ptr(), w2.numel(), _lib.ptr(plan.tile_counts_dev), _st())
        torch.cuda.synchronize()
        return dq, dkv, dkvr

    got = run()
    q64 = q.cpu().double().requires_grad_(True)
    kv64 = kv.cpu().double().requires_grad_(True)
    kvr64 = kvr.cpu().double().requires_grad_(True) if rte else None
    ref_agg, att_ref, _, _ = _edge_ref(plan, q64, kv64, kvr64, H)
    if hot:
        _check_hot(att_ref.detach())
    (ref_agg * dagg.cpu().double()).sum().backward()
    rows = plan.kv_rows
    errs = [_max_err(got[0].cpu(), q64.grad), _max_err(got[1][:rows].cpu(), kv64.grad[:rows])]
    if rte:
        errs.append(_max_err(got[2][:-1].cpu(), kvr64.grad[:-1]))
    assert max(errs) <= 5e-5, "max errors (dq, dkv[, dkvr]): %s" % ", ".join("%.3g" % e for e in errs)
    if det:
        again = run()
        for a, b in zip(got, again):
            if a is not None:
                assert torch.equal(a, b)
