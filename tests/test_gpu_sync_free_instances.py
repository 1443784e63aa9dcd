"""Every edge-kernel instance on sync-free plans, with everything past the device counts poisoned (run on an H100:
``pytest -m gpu``).

A sync-free plan (plan.build_plan(..., host_meta=...): to_torch(prebuild_plan=True), GraphedForward / GraphedTrainStep
replays, device batches of the GPU sampler) keeps {n_tiles, n_split, n_hubs} on the device (plan.tile_counts_dev); the
host fields are only the bounds the arrays were sized with (plan.tile_bounds), and so are those of every SourceIndex of
the deterministic row passes, whatever plan it comes from.  Every edge kernel therefore reads its tile count
(`p.d_counts ? p.d_counts[0] : p.n_tiles`) or hub count from the device, over a grid sized from the host bound.  The
slots past the device counts are torch.empty: in a training loop they hold an earlier batch's tiles.

Here they hold in-range poison instead (poison_tails; tests/test_sync_free_bounds_cpu.py checks that every entry
stays in range and that a consumer reading to the bound gets another answer):
  * copies of real tiles and hubs (a tile processed twice doubles an atomic gradient),
  * tiles that name a real destination with another destination's edge range, as whole rows and as hub pieces,
  * hub entries pointing at real slots with a wrong piece count, or at a real destination and an unused slot,
  * NaN in every partial slot of the workspaces (the used ones are overwritten).
Every result on the poisoned sync-free plans (type-sorted host_meta and not) must equal the synchronous plan's bitwise
(tiles come from an atomic counter and a tile's arithmetic does not depend on the grid), except the atomic backward,
which is compared with float64 like tests/test_gpu_edge_instances.py.

Deliberate faults, each built once into a temporary library (not committed) and run against this file on an H100
with -x; every one failed at the first case it reaches (FWD = test_forward_matches_synchronous_plan, BWD =
test_backward_matches_synchronous_plan, rel. error = max |got - float64| / max |float64|):

  fault: the host bound read where the device count belongs     first failure and what it saw
  k_edge_fwd_tma, n_tiles                                       FWD[d16-H4-2-fp32]: agg differs from the sync plan's
  k_edge_fwd_ldg, n_tiles                                       FWD[d16-H4-1-fp32]: agg differs
  k_merge_partials, n_hubs                                      FWD[d16-H4-1-fp32]: agg differs
  k_edge_bwd (atomic backward), n_tiles                         BWD[d16-H4-False-fp32]: dq, dkv rel. error 1.9e4, 1.1e4
  k_edge_bwd_dst, n_tiles                                       BWD[d16-H4-False-fp32]: deterministic dq rel. error 1.9e4
  k_edge_bwd_rows, n_tiles                                      BWD[d16-H4-False-fp32]: deterministic dkv rel. error 1e4
  k_merge_piece_rows, n_hubs                                    BWD[d16-H4-False-fp32]: deterministic dq, dkv NaN
  k_att_grad_prep, n_tiles                                      BWD[d16-H4-True-fp32]: dq, dkv rel. error 5.9, 5.8
  both hub merges read the hub list to n_hubs_host              FWD[d16-H4-1-fp32]: agg differs
"""
import bisect
import ctypes
import types

import pytest
import torch

from pyhgt_b200 import _lib, graphed, plan as P, synth, trim
from tests.test_gpu_att_grad import _deterministic
from tests.test_gpu_edge_instances import CASES, _dev, _edge_ref, _graph, _max_err, _q_scale, _st, _tables

T_, R_ = 3, 2
KINDS = ["fp32", "bf16", "t24"]


# ---------------------------------------------------------------------------------------------------------------------
# poison (device-agnostic: the CPU test runs it on CPU tensors)

def poison_tails(tiles, hubs, counts, bounds, ptr, seed=0):
    """Overwrite tiles[counts[0]:bounds[0]] and hubs[counts[2]:bounds[2]] with in-range entries that change a result if a
    kernel reads them.  counts / bounds: (n_tiles, n_split, n_hubs) as the device holds them / as the host sized the
    arrays; ptr: the row pointer the tiles cut (plan.row_ptr, or a SourceIndex's ptr).  Tiles cycle through a copy of a
    real tile, a hub piece of destination a over destination b's edges into a slot below the n_split bound, and a whole
    row a over the edges from an earlier row b with edges up to its own end; hubs through a copy of a real hub, a real
    hub with one piece fewer or more, and a non-hub row reading one slot past the used ones.  Returns the two lists
    written."""
    n_t, n_s, n_h = (int(c) for c in counts)
    b_t, b_s, b_h = (int(b) for b in bounds)
    ptr = ptr.cpu().long()
    n_rows = ptr.numel() - 1
    gen = torch.Generator().manual_seed(seed)

    def rnd(hi):
        return int(torch.randint(0, hi, (1,), generator=gen))

    real_t, real_h = tiles[:n_t].cpu(), hubs[:n_h].cpu()
    is_hub = torch.zeros(max(n_rows, 1), dtype=torch.bool)
    if n_h:
        is_hub[real_h[:, 0].long()] = True
    with_edges = (ptr[1:] > ptr[:-1]).nonzero().flatten().tolist()
    plain = (~is_hub[:n_rows]).nonzero().flatten().tolist()                    # rows a whole-row tile may name
    later = [a for a in plain if with_edges and a > with_edges[0]]
    t_rows = []
    for i in range(max(b_t - n_t, 0)):
        kind = i % 3
        if kind == 1 and b_s > 0 and n_rows:
            a, b = rnd(n_rows), rnd(n_rows)
            t_rows.append([a, -rnd(b_s) - 1, int(ptr[b]), int(ptr[b + 1])])
        elif kind == 2 and later:
            a = later[rnd(len(later))]
            b = with_edges[rnd(bisect.bisect_left(with_edges, a))]
            t_rows.append([a, a + 1, int(ptr[b]), int(ptr[a + 1])])
        elif n_t:
            t_rows.append(real_t[rnd(n_t)].tolist())
        else:
            a = rnd(n_rows)
            t_rows.append([a, a + 1, int(ptr[a]), int(ptr[a + 1])])
    h_rows = []
    for i in range(max(b_h - n_h, 0)):
        kind = i % 3
        if kind == 0 and n_h:
            h_rows.append(real_h[rnd(n_h)].tolist())
        elif kind == 1 and n_h:
            dst, s0, k = real_h[rnd(n_h), :3].tolist()
            k = k + 1 if i % 2 and s0 + k + 1 <= b_s else k - 1                # real hubs have at least 2 pieces
            h_rows.append([dst, s0, k, 0])
        else:
            a = plain[rnd(len(plain))] if plain else rnd(n_rows)
            h_rows.append([a, n_s + rnd(b_s - n_s), 1, 0])
    if t_rows:
        tiles[n_t:n_t + len(t_rows)] = torch.tensor(t_rows, dtype=torch.int32).to(tiles.device)
    if h_rows:
        hubs[n_h:n_h + len(h_rows)] = torch.tensor(h_rows, dtype=torch.int32).to(hubs.device)
    return t_rows, h_rows


def _counts(t):
    return [int(v) for v in t.cpu()[:3]]


def poison_plan(plan, seed, rte):
    """Poison a plan's tiles and hubs past its device counts (sync-free plans) and those of its source indices (every
    plan), built with CSR positions so that the att passes reuse them."""
    if plan.tile_counts_dev is not None:
        c = _counts(plan.tile_counts_dev)
        b = (plan.n_tiles, plan.n_split, plan.n_hubs)
        assert all(x <= y for x, y in zip(c, b)), (c, b)
        poison_tails(plan.tiles, plan.hubs, c, b, plan.row_ptr, seed)
    for which in (("kv", "rte") if rte else ("kv",)):
        idx = P.source_index(plan, which, with_pos=True)
        c = _counts(idx.counts_dev)
        b = (idx.n_tiles, idx.n_split, idx.n_hubs)
        assert all(x <= y for x, y in zip(c, b)), (which, c, b)
        poison_tails(idx.tiles, idx.hubs, c, b, idx.ptr, seed + 1 + len(which))


def _nan_ws(nbytes, dev):
    """A workspace whose partial slots (past the 256-byte counter block) hold NaN."""
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    if nbytes > 256:
        ws[256:].view(torch.float32).fill_(float("nan"))
    return ws


def _host_meta(g, T, R, sorted_):
    counts = torch.bincount(g.node_type, minlength=T)[:T].tolist()
    pairs = sorted({(int(s), int(r)) for s, r in zip(g.node_type[g.edge_index[0]].tolist(), g.edge_type.tolist())})
    return {"type_count": counts + [0], "sorted": sorted_, "pairs": pairs}


def _plans(g, rte, seed, T=T_, R=R_, meta=None):
    """The synchronous plan of graph g and its sync-free plans with type-sorted and unsorted host_meta, all poisoned."""
    dev = _dev()
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev) if rte else None, T, R)
    plans = [P.build_plan(*args)]
    if meta is not None:
        plans.append(P.build_plan(*args, host_meta=meta))
    else:
        sorted_ = bool((g.node_type[1:] >= g.node_type[:-1]).all())
        for s in ([True, False] if sorted_ else [False]):
            plans.append(P.build_plan(*args, host_meta=_host_meta(g, T, R, s)))
    for i, pl in enumerate(plans):
        poison_plan(pl, 100 * seed + i, rte)
    E = plans[0].n_edges
    for pl in plans[1:]:
        c = _counts(pl.tile_counts_dev)
        assert (c[0], c[1], c[2]) == (plans[0].n_tiles, plans[0].n_split, plans[0].n_hubs)
        assert torch.equal(pl.tiles[:c[0]], plans[0].tiles[:c[0]]) and torch.equal(pl.kv_row[:E], plans[0].kv_row[:E])
    return plans


def _sorted_graph(seed, **kw):
    g = _graph(T_, R_, seed=seed, **kw)
    g.node_type = g.node_type.sort().values
    return g


# ---------------------------------------------------------------------------------------------------------------------
# calls with poisoned workspaces

def _fwd(plan, q, kv, kvr, d, H, variant, kind, gelu=False, T=T_):
    """agg, att, stats, g_hi, g_lo of hgt_edge_forward[_bf16|_t24]."""
    dev = q.device
    N, E = plan.n_nodes, plan.n_edges
    agg = torch.full((N, d), float("nan"), device=dev)
    att = torch.full((max(E, 1), H), float("nan"), device=dev)
    stats = torch.full((N, 2 * H), float("nan"), device=dev)
    g_hi = torch.empty(N, d, dtype=torch.bfloat16, device=dev) if gelu else None
    g_lo = torch.empty(N, d, dtype=torch.bfloat16, device=dev) if gelu else None
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_workspace_bytes", plan.n_split, d, H, ctypes.byref(wsb))
    ws = _nan_ws(wsb.value, dev)
    fn = "hgt_edge_forward" + {"fp32": "", "bf16": "_bf16", "t24": "_t24"}[kind]
    _lib.call(fn, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
              plan.rte_row.data_ptr() if kvr is not None else None, plan.csr_eid.data_ptr(), plan.tiles.data_ptr(),
              plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, N, E, d, H, int(gelu), agg.data_ptr(),
              att.data_ptr(), stats.data_ptr(), _lib.ptr(g_hi), _lib.ptr(g_lo), ws.data_ptr(), ws.numel(), variant,
              _lib.ptr(plan.tile_counts_dev), plan.type_row0_dev.data_ptr(), T, None, _st())
    return agg, att[:E], stats, g_hi, g_lo


def _prep(plan, att, datt, H):
    """hgt_edge_att_grad_prep (autograd._att_grad_prep) with NaN partial slots: (datt in CSR order, C)."""
    dev = att.device
    datt_csr = torch.full((max(plan.n_edges, 1), H), float("nan"), device=dev)
    c_att = torch.full((plan.n_nodes, H), float("nan"), device=dev)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_att_grad_workspace_bytes", plan.n_split, H, ctypes.byref(wsb))
    ws = _nan_ws(wsb.value, dev)
    _lib.call("hgt_edge_att_grad_prep", att.data_ptr(), datt.data_ptr(), plan.csr_eid.data_ptr(), plan.row_ptr.data_ptr(),
              plan.tiles.data_ptr(), plan.n_tiles, plan.n_split, plan.hubs.data_ptr(), plan.n_hubs, plan.n_nodes, H,
              c_att.data_ptr(), datt_csr.data_ptr(), ws.data_ptr(), ws.numel(), _lib.ptr(plan.tile_counts_dev), _st())
    return datt_csr, c_att


def _bwd(plan, q, kv, kvr, agg, dagg, stats, d, H, det, kind, att_grad=None):
    """dq, d[K'|V'], d RTE of the atomic backward or of the destination + row passes (autograd._edge_backward_det with
    NaN partial slots); att_grad: (datt_csr, C) from _prep for the *_att calls."""
    dev = q.device
    N = plan.n_nodes
    sfx = "_bf16" if kind == "bf16" else ""
    asfx, extra = ("_att", (att_grad[0].data_ptr(), att_grad[1].data_ptr())) if att_grad is not None else ("", ())
    rte = kvr is not None
    dq = torch.full((N, d), float("nan"), device=dev)
    dkv = torch.full((plan.kv_rows + 1, 2 * d), float("nan"), device=dev)
    dkvr = torch.full(kvr.shape, float("nan"), device=dev) if rte else None
    st = _st()
    if not det:
        ws = torch.empty(256, dtype=torch.uint8, device=dev)
        _lib.call("hgt_edge_backward" + asfx + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(),
                  dagg.data_ptr(), stats.data_ptr(), *extra, plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
                  plan.rte_row.data_ptr() if rte else None, plan.tiles.data_ptr(), plan.n_tiles, N, d, H,
                  plan.kv_rows + 1, kvr.shape[0] if rte else 0, dq.data_ptr(), dkv.data_ptr(), _lib.ptr(dkvr),
                  ws.data_ptr(), ws.numel(), _lib.ptr(plan.tile_counts_dev), st)
        return dq, dkv, dkvr
    kvi = P.source_index(plan, "kv", True)
    rti = P.source_index(plan, "rte", True) if rte else None
    D = torch.full((N, H), float("nan"), device=dev)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_edge_backward_det_workspace_bytes", plan.n_split, max(kvi.n_split, rti.n_split if rti else 0), d,
              ctypes.byref(wsb))
    ws = _nan_ws(wsb.value, dev)
    _lib.call("hgt_edge_backward_dst" + asfx + sfx, q.data_ptr(), kv.data_ptr(), _lib.ptr(kvr), agg.data_ptr(),
              dagg.data_ptr(), stats.data_ptr(), *extra, plan.row_ptr.data_ptr(), plan.kv_row.data_ptr(),
              plan.rte_row.data_ptr() if rte else None, plan.tiles.data_ptr(), plan.n_tiles, plan.n_split,
              plan.hubs.data_ptr(), plan.n_hubs, N, d, H, dq.data_ptr(), D.data_ptr(), ws.data_ptr(), ws.numel(),
              _lib.ptr(plan.tile_counts_dev), st)
    passes = [(kv, kvr, kvi, plan.kv_rows + 1, dkv)] + ([(kvr, kv, rti, kvr.shape[0], dkvr)] if rte else [])
    for own, oth, idx, own_rows, grad in passes:
        ws[256:].view(torch.float32).fill_(float("nan"))
        src_oth = None if oth is None else idx.oth.data_ptr()
        pos = (att_grad[0].data_ptr(),) if att_grad is not None else ()
        pos2 = (idx.pos.data_ptr(),) if att_grad is not None else ()
        _lib.call("hgt_edge_backward_rows" + asfx + sfx, q.data_ptr(), dagg.data_ptr(), stats.data_ptr(), D.data_ptr(),
                  *pos, own.data_ptr(), _lib.ptr(oth), idx.ptr.data_ptr(), idx.dst.data_ptr(), src_oth, *pos2,
                  idx.n_rows, own_rows, idx.tiles.data_ptr(), idx.n_tiles, idx.n_split, idx.hubs.data_ptr(),
                  idx.n_hubs, d, H, grad.data_ptr(), ws.data_ptr(), ws.numel(), idx.counts_dev.data_ptr(), st)
    return dq, dkv, dkvr


# ---------------------------------------------------------------------------------------------------------------------
# checks shared by the instance tests and the count edge cases

def _tables_of(plan, d, rte, seed, kind, q_scale=1.0):
    """(q, kv, kvr) as the kernel reads them, and (kv, kvr) widened to float64 for the reference."""
    from tests.test_gpu_t24_tables import decode, encode_t
    q, kv, kvr = _tables(plan, d, rte, seed, torch.bfloat16 if kind == "bf16" else torch.float32, q_scale)
    if kind == "t24":
        kv, kvr = encode_t(kv), None if kvr is None else encode_t(kvr)
        wide = decode(kv, 2 * d), None if kvr is None else decode(kvr, 2 * d)
    else:
        wide = kv, kvr
    return q, kv, kvr, tuple(None if t is None else t.cpu().double() for t in wide)


def check_forward(plans, d, H, rte, kind, variants=(1, 2), seed=0, hot=False, rows=None):
    """Forward on every plan, bitwise against plans[0] (the gelu hi/lo output too where d % 8 == 0), and against float64
    on plans[0]'s tables.  rows: a bool mask of the destinations a trimmed view computes; only those are compared, and
    plans[0] (the whole plan) only against float64."""
    dev = _dev()
    q, kv, kvr, (kv64, kvr64) = _tables_of(plans[0], d, rte, seed, kind, _q_scale(d, H, hot))
    N, E = plans[0].n_nodes, plans[0].n_edges
    rp = plans[0].row_ptr.cpu().long()
    eid = plans[0].csr_eid[:E].cpu().long()
    rsel = torch.ones(N, dtype=torch.bool) if rows is None else rows
    esel = torch.repeat_interleave(rsel, rp[1:] - rp[:-1])              # CSR positions of the compared rows
    ssel = rsel & ((rp[1:] - rp[:-1]) > 0)                              # (m, l) exist for rows with in-edges
    ref_agg, ref_att, ref_m, ref_l = _edge_ref(plans[0], q.cpu().double(), kv64, kvr64, H)
    atol = 1e-4 if hot else 1e-5
    rsel_d, ssel_d, eids_d = rsel.to(dev), ssel.to(dev), eid[esel].to(dev)

    def view(o):
        agg, att, stats, hi, lo = o
        return (agg[rsel_d], att[eids_d], stats[ssel_d]) + tuple(None if t is None else t[rsel_d] for t in (hi, lo))

    bit = slice(None) if rows is None else slice(1, None)
    for variant in variants:
        for gelu in ((False, True) if d % 8 == 0 else (False,)):
            outs = [_fwd(pl, q, kv, kvr, d, H, variant, kind, gelu) for pl in plans]
            torch.cuda.synchronize()
            views = [view(o) for o in outs[bit]]
            for i, v in enumerate(views[1:], 1):
                for name, a, b in zip(("agg", "att", "stats", "g_hi", "g_lo"), v, views[0]):
                    if a is not None:
                        assert torch.equal(a, b), "plan %d, variant %d, gelu %s: %s differs" % (i, variant, gelu, name)
            want = torch.nn.functional.gelu(ref_agg) if gelu else ref_agg
            for i, (agg, att, stats, _, _) in enumerate(outs):
                agg, stats = agg.cpu().double(), stats.cpu().double()
                torch.testing.assert_close(agg[rsel], want[rsel], rtol=1e-4, atol=atol)
                torch.testing.assert_close(att.cpu().double()[eid][esel], ref_att[esel], rtol=1e-4, atol=1e-6)
                torch.testing.assert_close(stats[:, :H][ssel], ref_m[ssel], rtol=1e-5, atol=atol)
                torch.testing.assert_close(stats[:, H:][ssel], ref_l[ssel], rtol=1e-4, atol=1e-5)


def check_backward(plans, d, H, rte, kind, att, seed=0, hot=False, rows=None):
    """Atomic and deterministic backward (hgt_edge_att_grad_prep and the *_att calls when att) on every plan against
    float64 autograd of sum(agg * dagg) [+ sum(att * datt)] (<= 5e-5, as tests/test_gpu_edge_instances.py); the
    deterministic gradients bitwise equal across plans and on a second run.  rows: a bool mask of the destinations a
    trimmed view computes; dagg and datt are zero elsewhere, and plans[0] (the whole plan, whose rows are split into
    other pieces) is compared with float64 only."""
    dev = _dev()
    q, kv, kvr, (kv64, kvr64) = _tables_of(plans[0], d, rte, seed + 1, kind, _q_scale(d, H, hot))
    N, E = plans[0].n_nodes, plans[0].n_edges
    rp = plans[0].row_ptr.cpu().long()
    eid = plans[0].csr_eid[:E].cpu().long()
    gen = torch.Generator().manual_seed(seed + 2)
    dagg = torch.randn(N, d, generator=gen)
    datt = torch.randn(E, H, generator=gen)
    if rows is not None:
        dagg[~rows] = 0
        datt[eid[~torch.repeat_interleave(rows, rp[1:] - rp[:-1])]] = 0
    dagg, datt = dagg.to(dev), datt.to(dev)
    agg, att_t, stats = _fwd(plans[0], q, kv, kvr, d, H, 1, kind)[:3]

    q64 = q.cpu().double().requires_grad_(True)
    kv64 = kv64.clone().requires_grad_(True)
    kvr64 = kvr64.clone().requires_grad_(True) if rte else None
    ref_agg, ref_att, _, _ = _edge_ref(plans[0], q64, kv64, kvr64, H)
    loss = (ref_agg * dagg.cpu().double()).sum()
    if att:
        loss = loss + (ref_att * datt.cpu().double()[eid]).sum()
    loss.backward()
    want = (q64.grad, kv64.grad[:plans[0].kv_rows], kvr64.grad[:-1] if rte else None)

    def run(pl, det):
        return _bwd(pl, q, kv, kvr, agg, dagg, stats, d, H, det, kind, _prep(pl, att_t, datt, H) if att else None)

    det_runs = []
    for i, pl in enumerate(plans):
        for det in (False, True):
            got = run(pl, det)
            torch.cuda.synchronize()
            errs = [_max_err(got[0].cpu(), want[0]), _max_err(got[1][:pl.kv_rows].cpu(), want[1])]
            if rte:
                errs.append(_max_err(got[2][:-1].cpu(), want[2]))
            assert max(errs) <= 5e-5, "plan %d, det %s: max errors (dq, dkv[, dkvr]): %s" % (
                i, det, ", ".join("%.3g" % e for e in errs))
            if det and (rows is None or i > 0):
                det_runs.append(got)
    det_runs.append(run(plans[-1], True))
    torch.cuda.synchronize()
    for j, r in enumerate(det_runs[1:], 1):
        for name, a, b in zip(("dq", "dkv", "dkvr"), r, det_runs[0]):
            if a is not None:
                assert torch.equal(a, b), "deterministic %s: run %d differs from the first plan's" % (name, j)


# ---------------------------------------------------------------------------------------------------------------------
# 1. every instance

def _case_id(c):
    d, H, rte, hot = c
    return "d%d-H%d%s%s" % (d, H, "-rte" if rte else "", "-hot" if hot else "")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("d,H,rte,hot", CASES, ids=[_case_id(c) for c in CASES])
def test_forward_matches_synchronous_plan(d, H, rte, hot, variant, kind):
    """agg, att, stats and the gelu hi/lo output on the poisoned sync-free plans bitwise equal the synchronous plan's,
    and float64 at tests/test_gpu_edge_instances.py's tolerances."""
    if kind == "t24" and d % 8:
        pytest.skip("24-bit tables need d % 8 == 0")
    plans = _plans(_sorted_graph(d + H), rte, d + H)
    check_forward(plans, d, H, rte, kind, (variant,), seed=d, hot=hot)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fp32", "bf16"])
@pytest.mark.parametrize("att", [False, True])
@pytest.mark.parametrize("d,H,rte,hot", CASES, ids=[_case_id(c) for c in CASES])
def test_backward_matches_synchronous_plan(d, H, rte, hot, att, kind):
    """Atomic backward against float64 (<= 5e-5), deterministic dst + rows passes bitwise equal to the synchronous
    plan's and repeatable; att: hgt_edge_att_grad_prep and the *_att calls, both ways."""
    plans = _plans(_sorted_graph(2 * d + H), rte, 2 * d + H)
    check_backward(plans, d, H, rte, kind, att, seed=d, hot=hot)


# ---------------------------------------------------------------------------------------------------------------------
# 2. counts at their edges

def _run(plans, d, H, rte, rows=None):
    check_forward(plans, d, H, rte, "fp32", seed=d, rows=rows)
    for att in (False, True):
        check_backward(plans, d, H, rte, "fp32", att, seed=d, rows=rows)


@pytest.mark.gpu
def test_edges_above_split_without_a_hub():
    """E > TILE_SPLIT_EDGES but no destination above it: the device n_hubs is 0 while the bound (and the merge grid)
    is not."""
    g = synth.make_random(900, 6000, T_, R_, seed=5, sorted_types=True, self_loops=20)
    assert g.edge_index.shape[1] > P.TILE_SPLIT_EDGES
    plans = _plans(g, True, 5)
    assert plans[0].n_hubs == 0 and all(pl.n_hubs > 0 and pl.n_split > 0 for pl in plans[1:])
    _run(plans, 64, 4, True)


@pytest.mark.gpu
def test_more_hubs_than_the_merge_grid():
    """More hubs than 4 x SMs: k_merge_partials and k_merge_piece_rows stride over the hub list."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_hubs = 4 * sms + 37
    deg = P.TILE_SPLIT_EDGES + 1
    n = 2 * n_hubs + 300
    gen = torch.Generator().manual_seed(9)
    g = synth.make_random(n, 4000, T_, R_, seed=9, sorted_types=True, self_loops=20)
    hub_dst = torch.arange(n_hubs, dtype=torch.int64).repeat_interleave(deg) * 2
    src = torch.randint(0, n, (hub_dst.numel(),), generator=gen)
    g.edge_index = torch.cat([g.edge_index, torch.stack([src, hub_dst])], 1)
    g.edge_type = torch.cat([g.edge_type, torch.randint(0, R_, (hub_dst.numel(),), generator=gen)])
    g.edge_time = torch.cat([g.edge_time, torch.randint(0, 240, (hub_dst.numel(),), generator=gen)])
    plans = _plans(g, False, 9)
    assert plans[0].n_hubs >= n_hubs > 4 * sms
    check_forward(plans, 32, 8, False, "fp32", seed=3)
    check_backward(plans, 32, 8, False, "fp32", True, seed=3)


@pytest.mark.gpu
def test_no_edges():
    """N > 0 with E = 0: tile bounds above zero, no hub, nothing to gather."""
    g = synth.make_random(500, 0, T_, R_, seed=2, sorted_types=True)
    assert g.edge_index.shape[1] == 0
    plans = _plans(g, True, 2, meta=_host_meta(g, T_, R_, True))
    assert plans[1].n_tiles > 0 and plans[1].n_split == 0
    dev = _dev()
    d, H = 64, 4
    q, kv, kvr = _tables(plans[0], d, True, 1, torch.float32)
    for variant in (1, 2):
        outs = [_fwd(pl, q, kv, kvr, d, H, variant, "fp32") for pl in plans]
        for o in outs:
            assert torch.equal(o[0], torch.zeros(plans[0].n_nodes, d, device=dev))
    dagg = torch.randn(plans[0].n_nodes, d, device=dev)
    agg, _, stats = outs[0][:3]
    for pl in plans:
        for det in (False, True):
            got = _bwd(pl, q, kv, kvr, agg, dagg, stats, d, H, det, "fp32")
            assert all(torch.equal(t, torch.zeros_like(t)) for t in got)


@pytest.mark.gpu
def test_signature_padded_batch():
    """A batch padded to a GraphSignature (graphed.pad_batch): the bounds come from the signature and sit far above the
    counts; the padding edges all enter the pad node, which becomes a hub."""
    T, R = T_, R_
    b = synth.make_random(400, 3000, T, R, seed=11, sorted_types=True, self_loops=20)
    counts = [int((b.node_type == t).sum()) + 150 for t in range(T)]
    pairs = {(int(b.node_type[s]), int(r)) for s, r in zip(b.edge_index[0].tolist(), b.edge_type.tolist())}
    sig = graphed.GraphSignature(counts, 9000, pairs, R, 8, use_time=True)
    x, nt, tm, ei, et, _ = graphed.pad_batch(sig, torch.zeros(400, 8), b.node_type, b.edge_time, b.edge_index,
                                             b.edge_type)
    g = types.SimpleNamespace(node_type=torch.as_tensor(nt), edge_index=torch.as_tensor(ei),
                              edge_type=torch.as_tensor(et), edge_time=torch.as_tensor(tm))
    plans = _plans(g, True, 11, meta=sig.host_meta())
    c = _counts(plans[1].tile_counts_dev)
    assert plans[1].n_tiles > c[0] + 50 and plans[1].n_hubs > c[2]
    _run(plans, 64, 4, True)


@pytest.mark.gpu
def test_trimmed_range_tiles():
    """Tiles over destination row ranges (hgt_plan_range_tiles, trim._range_view), poisoned like the others: the rows
    inside the ranges equal the whole plan's bitwise, and the masked source indices give the float64 gradients of a
    loss on those rows."""
    g = _sorted_graph(13)
    full = _plans(g, True, 13)[0]
    N = full.n_nodes
    ranges = [(0, 40), (100, 101), (250, 520), (800, N)]
    view = trim._range_view(full, ranges)
    poison_plan(view, 1300, True)
    rows = torch.zeros(N, dtype=torch.bool)
    for a, b in ranges:
        rows[a:b] = True
    assert rows[3]                                           # the hub destination of _graph lies inside
    _run([full, view], 64, 4, True, rows=rows)


# ---------------------------------------------------------------------------------------------------------------------
# 3. one layer

@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "bf16", "no_grad"])
def test_layer_on_poisoned_sync_free_plan(mode):
    """HGTConv on a poisoned sync-free plan (type-sorted host_meta and not): the forward, and for the training modes
    the deterministic step's input and parameter gradients, bitwise equal the synchronous plan's.  fp32 tables,
    bf16 autocast, and the no-grad forward on 24-bit tables."""
    import pyhgt_b200
    dev = _dev()
    d, H = 64, 4
    g = _sorted_graph(17)
    torch.manual_seed(0)
    m = pyhgt_b200.HGTConv(d, d, T_, R_, H, 0.0, True, True).to(dev)
    x = torch.randn(g.node_type.numel(), d, generator=torch.Generator().manual_seed(1)).to(dev)
    args = (g.node_type.to(dev), g.edge_index.to(dev), g.edge_type.to(dev), g.edge_time.to(dev))
    w = torch.randn(g.node_type.numel(), d, generator=torch.Generator().manual_seed(2)).to(dev)
    results = []
    for i, meta in enumerate((None, _host_meta(g, T_, R_, True), _host_meta(g, T_, R_, False))):
        P.clear_plan_cache()
        pl = P.get_plan(*args, T_, R_, host_meta=meta)
        poison_plan(pl, 1700 + i, True)
        m.zero_grad(set_to_none=True)
        if mode == "no_grad":
            with torch.no_grad():
                results.append((m(x, *args),))
            continue
        xg = x.clone().requires_grad_(True)
        with _deterministic(True), torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
            out = m(xg, *args)
            (out.float() * w).sum().backward()
        results.append((out.detach(), xg.grad) + tuple(p.grad.clone() for p in m.parameters() if p.grad is not None))
    P.clear_plan_cache()
    for i, r in enumerate(results[1:], 1):
        assert len(r) == len(results[0])
        for j, (a, b) in enumerate(zip(r, results[0])):
            assert torch.equal(a, b), "plan %d, tensor %d differs from the synchronous plan's" % (i, j)
