"""Trimmed GNN forward, GNN.forward(..., out_nodes=) (pyhgt_b200/trim.py): hop distances and the hop order, edge tiles
over destination row ranges, and forward / training / deterministic / bf16 parity with the untrimmed forward's rows.

What each deliberate fault is caught by:
  hops one short (L - 1 BFS passes)                           test_hop_distances_and_order_match_numpy_bfs
  tiles crossing a range end (k_tile_close without end_of)    test_range_tiles_write_only_their_destinations
  the unmasked source index in the deterministic row pass     test_deterministic_trimmed_steps_are_bitwise_equal_and_finite
  kv_runs one hop short (K'/V' prefix dist <= L - l)          test_trimmed_forward_matches_full_rows
  a leaked unwritten row (torch.empty layer output)           test_trimmed_training_gradients_match_full,
                                                              test_deterministic_trimmed_steps_are_bitwise_equal_and_finite
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, plan as P, synth, trim   # noqa: E402
from tests.conftest import load_golden                # noqa: E402

FWD_MAX_ABS = 1e-5
GRAD_REL_FRO = 1e-4


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _graph(T=3, R=4, n=700, e=3500, seed=0, hub_in=(), hub_out=()):
    """make_random with unsorted types, isolated nodes, self loops, multi-edges, two nodes of unknown type (T and -1) and
    hub destinations: hub_in / hub_out = [(node, in-degree)]."""
    g = synth.make_random(n, e, T, R, seed=seed, isolated_frac=0.2, self_loops=25, duplicate_edges=60)
    nt = g.node_type.clone()
    nt[3], nt[11] = T, -1
    gen = torch.Generator().manual_seed(seed + 1)
    ei, et, tm = [g.edge_index], [g.edge_type], [g.edge_time]
    for v, deg in tuple(hub_in) + tuple(hub_out):
        ei.append(torch.stack([torch.randint(0, n, (deg,), generator=gen), torch.full((deg,), v)]))
        et.append(torch.randint(0, R, (deg,), generator=gen))
        tm.append(torch.randint(0, 240, (deg,), generator=gen))
    return nt, torch.cat(ei, 1), torch.cat(et), torch.cat(tm)


def _to(dev, *ts):
    return [t.to(dev) for t in ts]


def _np_dist(ei, N, seeds, L):
    dist = np.full(N, L + 1, dtype=np.int64)
    dist[np.asarray(seeds)] = 0
    src, dst = ei
    for h in range(1, L + 1):
        hit = src[dist[dst] == h - 1]
        dist[hit[dist[hit] > h]] = h
    return dist


def _gnn(T, R, L, rte=True, norm=True, F_in=32, d=64, H=4, dropout=0.0, seed=0):
    from pyhgt_b200.model import GNN
    torch.manual_seed(seed)
    m = GNN(F_in, d, T, R, H, L, dropout, "hgt", norm, norm, rte)
    with torch.no_grad():                                  # move the gates and priors off their initial constants
        for name, p in m.named_parameters():
            if name.endswith(("skip", "relation_pri")):
                p.add_(0.3 * torch.randn_like(p))
    return m.to(_dev())


def _seeds(N, k, seed):
    rng = np.random.RandomState(seed)
    s = rng.choice(N, k, replace=False)
    return np.concatenate([s, s[:3]])                     # duplicates, in no particular order


# ---------------------------------------------------------------------------------------------------------------------
# 1. hop distances and hop order

@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_hop_distances_and_order_match_numpy_bfs(L):
    dev = _dev()
    T, R = 3, 4
    nt, ei, et, tm = _graph(T, R, hub_in=[(5, 1300)])
    N = nt.numel()
    seeds = _seeds(N, 12, L)
    on = torch.from_numpy(seeds).to(dev)
    lay = trim.build_layout(*_to(dev, nt, ei, et, tm), on, T, R, L)
    dist = _np_dist(ei.numpy(), N, seeds, L)
    assert np.array_equal(lay.dist.cpu().numpy(), dist)
    ntn = nt.numpy()
    known = (ntn >= 0) & (ntn < T)
    key = np.where(known, np.clip(ntn, 0, T - 1) * (L + 2) + dist, T * (L + 2))
    perm = np.argsort(key, kind="stable")
    assert np.array_equal(lay.perm.cpu().numpy(), perm)                        # stable (type, hop) order
    rank = np.empty(N, dtype=np.int64)
    rank[perm] = np.arange(N)
    assert np.array_equal(lay.out_rows.cpu().numpy(), rank[seeds])
    for t in range(T):
        for b in range(L + 2):
            assert lay.counts[t, b] == int(((ntn == t) & (dist == b)).sum()), (t, b)
        s_t = np.unique(seeds[ntn[seeds] == t])                                  # seeds first, in original order
        r0 = lay.plan.type_row0[t]
        assert np.array_equal(perm[r0:r0 + s_t.size], s_t)
    full = P.get_plan(*_to(dev, nt, ei, et, tm), T, R)
    assert lay.plan.type_count == full.type_count and lay.plan.pairs == full.pairs
    assert lay.plan.sorted_types
    for l, view in enumerate(lay.layers, 1):                                   # per-layer prefixes from the counts
        assert view.active == tuple(int(lay.counts[t, :L - l + 1].sum()) for t in range(T))


# ---------------------------------------------------------------------------------------------------------------------
# 2. edge tiles over row ranges

def test_range_tiles_write_only_their_destinations():
    dev = _dev()
    T, R, d, H = 3, 4, 64, 4
    nt0 = _graph(T, R, seed=3)[0].numpy()                                      # rank order depends on node_type only
    perm = np.argsort(np.where((nt0 >= 0) & (nt0 < T), nt0, T), kind="stable")
    row0 = np.concatenate([[0], np.cumsum([(nt0 == t).sum() for t in range(T)])])
    ranges = [(int(row0[t] + (row0[t + 1] - row0[t]) // 4), int(row0[t] + (row0[t + 1] - row0[t]) // 2)) for t in range(T)]
    hub_in, hub_out = int(perm[ranges[0][0] + 1]), int(perm[ranges[1][1] + 2])
    nt, ei, et, tm = _graph(T, R, seed=3, hub_in=[(hub_in, 1500)], hub_out=[(hub_out, 1300)])
    nt, ei, et = _to(dev, nt, ei, et)
    pl = P.build_plan(nt, ei, et, None, T, R)
    rk = pl.rank.cpu().long()
    r5, r9 = int(rk[hub_in]), int(rk[hub_out])
    assert pl.n_hubs == 2
    view = trim._range_view(pl, ranges)
    N, E = pl.n_nodes, pl.n_edges
    g = torch.Generator(device=dev).manual_seed(0)
    q = torch.randn(N, d, device=dev, generator=g)
    kv = torch.randn(pl.kv_rows + 1, 2 * d, device=dev, generator=g)
    kv[-1].zero_()

    def run(p, fill):
        agg = torch.full((N, d), fill, device=dev)
        att = torch.full((E, H), fill, device=dev)
        stats = torch.full((N, 2 * H), fill, device=dev)
        wsb = ctypes.c_size_t()
        _lib.call("hgt_edge_workspace_bytes", p.n_split, d, H, ctypes.byref(wsb))
        ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
        _lib.call("hgt_edge_forward", q.data_ptr(), kv.data_ptr(), None, p.row_ptr.data_ptr(), p.kv_row.data_ptr(), None,
                  p.csr_eid.data_ptr(), p.tiles.data_ptr(), p.n_tiles, p.n_split, p.hubs.data_ptr(), p.n_hubs, N, E, d, H,
                  0, agg.data_ptr(), att.data_ptr(), stats.data_ptr(), None, None, ws.data_ptr(), ws.numel(), 0,
                  _lib.ptr(p.tile_counts_dev), None, 0, None, _st())
        return agg, att, stats

    full = run(pl, 0.0)
    part = run(view, 12345.0)
    inside = torch.zeros(N, dtype=torch.bool, device=dev)
    for a, b in ranges:
        inside[a:b] = True
    assert bool(inside[r5]) and not bool(inside[r9])
    rp = pl.row_ptr.long()
    e_dst = torch.repeat_interleave(torch.arange(N, device=dev), rp[1:] - rp[:-1])
    e_in = torch.zeros(E, dtype=torch.bool, device=dev)
    e_in[pl.csr_eid.long()] = inside[e_dst]
    for what, f, p_, sel in (("agg", full[0], part[0], inside), ("att", full[1], part[1], e_in),
                             ("stats", full[2], part[2], inside)):
        assert bool((p_[~sel] == 12345.0).all()), "%s: a row outside the ranges was written" % what
        assert torch.allclose(p_[sel], f[sel], rtol=0, atol=1e-6), "%s: rows inside the ranges differ" % what


# ---------------------------------------------------------------------------------------------------------------------
# 3. forward parity

def _fwd(m, x, nt, tm, ei, et, s):
    with torch.no_grad():
        return m(x, nt, tm, ei, et)[s], m(x, nt, tm, ei, et, out_nodes=s)


@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("rte", [True, False])
@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_trimmed_forward_matches_full_rows(L, rte, norm):
    """Observed on an H100: trimmed and full rows are bitwise equal, fused and per-stage alike."""
    import pyhgt_b200
    dev = _dev()
    T, R = 3, 4
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=L, hub_in=[(5, 1200)]))
    N = nt.numel()
    m = _gnn(T, R, L, rte, norm).eval()
    x = torch.randn(N, 32, device=dev)
    s = torch.from_numpy(_seeds(N, 16, L + 10)).to(dev)
    s[0] = 3                                                                    # a node of unknown type: zero row
    for fused in (True, False):
        pyhgt_b200.HGTConv.fused_call = fused
        try:
            ref, got = _fwd(m, x, nt, tm, ei, et, s)
        finally:
            pyhgt_b200.HGTConv.fused_call = True
        assert got.shape == ref.shape
        err = (got - ref).abs().max().item()
        assert err <= FWD_MAX_ABS, "L=%d rte=%s norm=%s fused=%s: max abs %.3g" % (L, rte, norm, fused, err)
        assert bool((got[0] == 0).all())
    assert all(gc.base_conv.att is None for gc in m.gcs)


def _sampled_members(B, depth, width, seed=0):
    from pyhgt_b200 import sampler
    from tests.test_gpu_sampler_batched import _graph as _sgraph
    fx, fg, dg, _ = _sgraph("sampler")
    rng = np.random.RandomState(seed)
    inps = []
    for _ in range(B):
        ids = rng.choice(fg.n_ids["paper"], 12, replace=False)
        inps.append({"paper": np.stack([ids, rng.randint(2000, 2016, 12)], 1)})
    members = sampler.sample_subgraphs_cuda(dg, fx["time_range"], depth, width, inps,
                                            torch.Generator().manual_seed(seed))
    T, R = len(dg.types), len(dg.edge_dict)
    seeds = []
    for mb in members:
        p0 = P.get_plan(mb[1], mb[3], mb[4], mb[2], T, R).type_row0[dg.slot["paper"]]
        seeds.append(torch.arange(p0, p0 + 12, device=mb[1].device))
    return members, seeds, T, R


@pytest.mark.parametrize("L", [2, 3])
def test_trimmed_forward_on_sampled_batches_and_their_union(L):
    from pyhgt_b200 import sampler
    members, seeds, T, R = _sampled_members(3, 3, 8)
    m = _gnn(T, R, L, F_in=8).eval()
    for mb, s in zip(members, seeds):
        ref, got = _fwd(m, mb[0], mb[1], mb[2], mb[3], mb[4], s)
        assert (got - ref).abs().max().item() <= FWD_MAX_ABS
    nf, nt, tm, ei, et, rows = sampler.merge_batches(members, T, R)
    s = torch.cat([r.to(nt.device)[s_] for r, s_ in zip(rows, seeds)])
    ref, got = _fwd(m, nf, nt, tm, ei, et, s)
    assert (got - ref).abs().max().item() <= FWD_MAX_ABS


def test_trimmed_golden_gnn_rows_match_reference():
    from pyhgt_b200.model import GNN
    dev = _dev()
    fx = load_golden("gnn_2layer")
    c = fx["cfg"]
    m = GNN(c["in_dim"], c["n_hid"], c["num_types"], c["num_relations"], c["n_heads"], c["n_layers"], 0.2, "hgt",
            c["prev_norm"], c["last_norm"], c["use_RTE"])
    m.load_state_dict(fx["state_dict"], strict=True)
    m = m.to(dev).eval()
    s = torch.from_numpy(np.random.RandomState(0).choice(fx["node_type"].numel(), 20, replace=False)).to(dev)
    with torch.no_grad():
        got = m(fx["node_feature"].to(dev), fx["node_type"].to(dev), fx["edge_time"].to(dev), fx["edge_index"].to(dev),
                fx["edge_type"].to(dev), out_nodes=s)
    ref = fx["out"][s.cpu()]
    assert torch.allclose(got.cpu(), ref, rtol=1e-3, atol=1e-3), (got.cpu() - ref).abs().max().item()


# ---------------------------------------------------------------------------------------------------------------------
# 4. training parity, 5. deterministic steps

def _rel(got, ref):
    return float((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-30))


def _grads(m, x, nt, tm, ei, et, s, w, trimmed):
    m.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    out = m(xg, nt, tm, ei, et, out_nodes=s) if trimmed else m(xg, nt, tm, ei, et)[s]
    (out * w).sum().backward()
    return {"node_feature": xg.grad, **{n: p.grad for n, p in m.named_parameters()}}


@pytest.mark.parametrize("rte", [True, False])
@pytest.mark.parametrize("L", [2, 3])
def test_trimmed_training_gradients_match_full(L, rte):
    dev = _dev()
    T, R = 3, 4
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=20 + L, hub_in=[(5, 1200)]))
    N = nt.numel()
    m = _gnn(T, R, L, rte).train()
    x = torch.randn(N, 32, device=dev)
    s = torch.from_numpy(_seeds(N, 16, L)).to(dev)
    w = torch.randn(s.numel(), 64, device=dev)
    ref = _grads(m, x, nt, tm, ei, et, s, w, False)
    got = _grads(m, x, nt, tm, ei, et, s, w, True)
    for k in ref:
        if ref[k] is None:
            assert got[k] is None or not bool(got[k].any()), k
            continue
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], ref[k]) <= GRAD_REL_FRO, "%s: rel fro %.3g" % (k, _rel(got[k], ref[k]))


def test_deterministic_trimmed_steps_are_bitwise_equal_and_finite():
    dev = _dev()
    T, R, L = 3, 4, 3
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=31, hub_in=[(5, 2100)], hub_out=[(9, 1500)]))
    N = nt.numel()
    m = _gnn(T, R, L).train()
    x = torch.randn(N, 32, device=dev)
    s = torch.from_numpy(_seeds(N, 10, 4)).to(dev)
    w = torch.randn(s.numel(), 64, device=dev)
    with _deterministic(True):
        a = _grads(m, x, nt, tm, ei, et, s, w, True)
        b = _grads(m, x, nt, tm, ei, et, s, w, True)
    ref = _grads(m, x, nt, tm, ei, et, s, w, False)
    for k in a:
        if a[k] is None:
            continue
        assert torch.isfinite(a[k]).all(), k
        assert torch.equal(a[k], b[k]), k
        assert _rel(a[k], ref[k]) <= GRAD_REL_FRO, "%s: rel fro %.3g" % (k, _rel(a[k], ref[k]))


# ---------------------------------------------------------------------------------------------------------------------
# 6. bf16 autocast, 7. synchronisation and errors

def test_trimmed_forward_under_bf16_autocast_matches_full():
    dev = _dev()
    T, R, L = 3, 4, 3
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=41))
    N = nt.numel()
    m = _gnn(T, R, L).eval()
    x = torch.randn(N, 32, device=dev)
    s = torch.from_numpy(_seeds(N, 16, 5)).to(dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ref, got = _fwd(m, x, nt, tm, ei, et, s)
    assert (got - ref).abs().max().item() <= FWD_MAX_ABS


def test_cached_layout_runs_without_sync_and_errors():
    from pyhgt_b200.model import GNN
    dev = _dev()
    T, R, L = 3, 4, 2
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=51))
    N = nt.numel()
    m = _gnn(T, R, L).train()
    x = torch.randn(N, 32, device=dev)
    s = torch.arange(0, 40, 3, device=dev)
    m(x, nt, tm, ei, et, out_nodes=s).sum().backward()                        # builds and caches the layout
    with torch.no_grad():
        m(x, nt, tm, ei, et, out_nodes=s)                                      # and the inference path's pointer tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m(x, nt, tm, ei, et, out_nodes=s).sum().backward()
        with torch.no_grad():
            m(x, nt, tm, ei, et, out_nodes=s)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    with torch.no_grad():
        with pytest.raises(IndexError):
            m(x, nt, tm, ei, et, out_nodes=torch.tensor([0, N], device=dev))
        with pytest.raises(IndexError):
            m(x, nt, tm, ei, et, out_nodes=torch.tensor([-1], device=dev))
        out = m(x, nt, tm, ei, et, out_nodes=torch.empty(0, dtype=torch.int64, device=dev))
        assert tuple(out.shape) == (0, 64)
        with pytest.raises(_lib.HgtError):
            m(x.cpu(), nt.cpu(), tm.cpu(), ei.cpu(), et.cpu(), out_nodes=s.cpu())
        with pytest.raises(_lib.HgtError):
            m(x, nt, tm, ei, et, out_nodes=s.cpu())
        dense = GNN(32, 64, T, R, 4, 2, 0.0, "dense_hgt").to(dev).eval()
        with pytest.raises(ValueError):
            dense(x, nt, tm, ei, et, out_nodes=s)
