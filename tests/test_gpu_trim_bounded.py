"""Trimmed forwards from host-known hop bounds (trim.TrimSignature, hgt_trim_layout_bounded): the bounded layout against
hgt_trim_layout, padded trimmed rows against the exact ones, sync-free layouts of new batches, overflow handling, and the
trimmed forward and training step captured in CUDA graphs (graphed.py)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, graphed, plan as P, trim   # noqa: E402
from tests.test_gpu_trim import (FWD_MAX_ABS, _deterministic, _dev, _gnn, _graph, _rel,  # noqa: E402
                                 _sampled_members, _seeds, _to)

PADDED_GRAD_REL_FRO = 4e-6   # padded against exact trimmed gradients
# Graphed trimmed against graphed untrimmed gradients: the trimmed backward sums dW / bias over fewer rows and in other
# groups, so the two differ by fp32 rounding.  An H100 run measured 6.0e-6 for the worst parameter, which does not hold
# 4e-6; the bar keeps a 3x margin, well inside test_gpu_trim.py's 1e-4 for trimmed against full gradients.
GRAPHED_GRAD_REL_FRO = 2e-5
BF16_GRAD_REL_FRO = 5e-2     # test_gpu_bf16_tables.py's bound for bf16-table gradients
CANARY = -7


def _layout(nt, ei, et, tm, on, T, R, L, bounds=None, n_rows=None, spare=64):
    """One call of hgt_trim_layout (bounds None) or hgt_trim_layout_bounded, with canaries past the ends of the
    row-indexed outputs.  Returns numpy copies of every output."""
    dev = nt.device
    N, E, n_out = nt.numel(), ei.shape[1], on.numel()
    n_rows = N if n_rows is None else n_rows
    n_counts = T * (L + 2)
    i32 = dict(dtype=torch.int32, device=dev)
    i64 = dict(dtype=torch.int64, device=dev)
    wsb = ctypes.c_size_t()
    _lib.call("hgt_plan_workspace_bytes", N, E, ctypes.byref(wsb))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    dist = torch.full((N,), CANARY, **i32)
    perm = torch.full((n_rows + spare,), CANARY, **i32)
    rank = torch.full((N,), CANARY, **i32)
    hnt = torch.full((n_rows + spare,), CANARY, **i64)
    hei = torch.full((2, E), CANARY, **i64)
    rows = torch.full((n_out,), CANARY, **i64)
    meta = torch.full((2 * n_counts + T * R + 6,), CANARY, **i32)
    args = (nt.data_ptr(), N, E, T, R, on.data_ptr(), n_out, L)
    outs = (dist.data_ptr(), perm.data_ptr(), rank.data_ptr(), hnt.data_ptr(), hei.data_ptr(), rows.data_ptr(),
            meta.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    if bounds is None:
        _lib.call("hgt_trim_layout", ei.data_ptr(), et.data_ptr(), _lib.ptr(tm), *args, *outs)
    else:
        b = np.ascontiguousarray(bounds, dtype=np.int32)
        _lib.call("hgt_trim_layout_bounded", ei.data_ptr(), et.data_ptr(), _lib.ptr(tm), *args, b.ctypes.data, n_rows,
                  *outs)
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in dict(dist=dist, perm=perm, rank=rank, nt=hnt, ei=hei, rows=rows).items()}
    m = meta.cpu().numpy()
    r["counts"] = m[:n_counts].reshape(T, L + 2)
    r["head"] = m[:n_counts + T * R + 4]
    r["flags"] = m[n_counts + T * R:n_counts + T * R + 4]
    r["off"] = m[n_counts + T * R + 4:]
    return r


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact bounds: hgt_trim_layout's layout, bitwise

@pytest.mark.parametrize("L", [1, 2, 4])
def test_exact_bounds_reproduce_the_read_back_layout(L):
    dev = _dev()
    T, R = 3, 4
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=60 + L, hub_in=[(5, 1300)]))      # two nodes of unknown type
    N = nt.numel()
    on = torch.from_numpy(_seeds(N, 12, L)).to(dev)
    ref = _layout(nt, ei, et, tm, on, T, R, L)
    got = _layout(nt, ei, et, tm, on, T, R, L, bounds=ref["counts"], n_rows=N)
    for k in ("dist", "perm", "rank", "nt", "ei", "rows", "head"):
        assert np.array_equal(got[k], ref[k]), k
    assert (ref["perm"][N:] == CANARY).all() and (got["perm"][N:] == CANARY).all()
    assert not got["flags"].any()
    c = ref["counts"].reshape(-1)
    assert np.array_equal(got["off"], np.concatenate([[0], np.cumsum(c), [N]]))
    # the read-back build itself runs on the same placement: its layout is the exact-bounds one
    lay = trim.build_layout(nt, ei, et, tm, on, T, R, L)
    assert np.array_equal(lay.perm.cpu().numpy(), ref["perm"][:N]) and np.array_equal(lay.bounds, ref["counts"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. slack bounds: padded trimmed rows equal the exact trimmed rows

def _fwd3(m, x, nt, tm, ei, et, s, tsig):
    with torch.no_grad():
        return (m(x, nt, tm, ei, et)[s], m(x, nt, tm, ei, et, out_nodes=s),
                m(x, nt, tm, ei, et, out_nodes=s, trim_signature=tsig))


@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("rte", [True, False])
@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_slack_bounds_match_exact_trimmed_and_full_rows(L, rte, norm):
    import pyhgt_b200
    dev = _dev()
    T, R = 3, 4
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=L, hub_in=[(5, 1200)]))
    N = nt.numel()
    m = _gnn(T, R, L, rte, norm).eval()
    x = torch.randn(N, 32, device=dev)
    s = torch.from_numpy(_seeds(N, 16, L + 10)).to(dev)
    s[0] = 3                                                                    # a node of unknown type: zero row
    tsig = trim.TrimSignature.for_batches([(x, nt, tm, ei, et)], [s], L, 0.3, num_types=T, num_relations=R)
    assert (tsig.hop_bounds[:, L + 1] == 0).all()
    for fused in (True, False):
        pyhgt_b200.HGTConv.fused_call = fused
        try:
            full, exact, padded = _fwd3(m, x, nt, tm, ei, et, s, tsig)
        finally:
            pyhgt_b200.HGTConv.fused_call = True
        assert torch.equal(padded, exact), "L=%d rte=%s norm=%s fused=%s" % (L, rte, norm, fused)
        assert (padded - full).abs().max().item() <= FWD_MAX_ABS
        assert bool((padded[0] == 0).all())
    lay = trim.get_layout(nt, ei, et, tm if rte else None, s, T, R, L, tsig, P.get_plan(nt, ei, et, tm, T, R).pairs)
    lay.check()
    assert lay.plan.n_nodes == int(tsig.hop_bounds.sum()) + 1


@pytest.mark.parametrize("L", [2, 3])
def test_slack_bounds_on_sampled_batches_and_their_union(L):
    from pyhgt_b200 import sampler
    members, seeds, T, R = _sampled_members(3, 3, 8)
    m = _gnn(T, R, L, F_in=8).eval()
    tsig = trim.TrimSignature.for_batches(members, seeds, L, 0.1, num_types=T, num_relations=R)
    for mb, s in zip(members, seeds):
        full, exact, padded = _fwd3(m, *mb[:5], s, tsig)
        assert torch.equal(padded, exact)
        assert (padded - full).abs().max().item() <= FWD_MAX_ABS
    nf, nt, tm, ei, et, rows = sampler.merge_batches(members, T, R)
    s = torch.cat([r.to(nt.device)[s_] for r, s_ in zip(rows, seeds)])
    usig = trim.TrimSignature.for_batches([(nf, nt, tm, ei, et)], [s], L, 0.1, num_types=T, num_relations=R)
    full, exact, padded = _fwd3(m, nf, nt, tm, ei, et, s, usig)
    assert torch.equal(padded, exact)
    assert (padded - full).abs().max().item() <= FWD_MAX_ABS


# ---------------------------------------------------------------------------------------------------------------------
# 3. a new batch with a signature: forward and backward without a host sync

@pytest.mark.parametrize("det", [False, True])
def test_new_batch_with_signature_trains_without_sync(det):
    L = 3
    members, seeds, T, R = _sampled_members(4, 3, 8, seed=5)
    tsig = trim.TrimSignature.for_batches(members, seeds, L, 0.2, num_types=T, num_relations=R)
    m = _gnn(T, R, L, F_in=8).train()
    w = torch.randn(seeds[0].numel(), 64, device=seeds[0].device)
    with _deterministic(det):
        m(*members[0][:5], out_nodes=seeds[0], trim_signature=tsig).mul(w).sum().backward()   # warm-up: pointer tables
        torch.cuda.synchronize()
        grads = []
        for mb, s in zip(members[1:], seeds[1:]):                                # batches never seen by the layout cache
            m.zero_grad(set_to_none=False)
            torch.cuda.set_sync_debug_mode("error")
            try:
                m(*mb[:5], out_nodes=s, trim_signature=tsig).mul(w).sum().backward()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            grads.append([p.grad.clone() for p in m.parameters()])
            ref = [g.clone() for g in grads[-1]]
            m.zero_grad(set_to_none=False)
            m(*mb[:5], out_nodes=s).mul(w).sum().backward()                      # exact trimmed step
            for g, p in zip(ref, m.parameters()):
                assert torch.isfinite(g).all()
                assert _rel(g, p.grad) <= PADDED_GRAD_REL_FRO
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# 4. overflow and out-of-range ids

def test_overflow_writes_no_row_past_its_region_and_yields_nan():
    dev = _dev()
    T, R, L = 3, 4, 2
    nt, ei, et, tm = _to(dev, *_graph(T, R, seed=71))
    N = nt.numel()
    on = torch.from_numpy(_seeds(N, 12, 3)).to(dev)
    exact = _layout(nt, ei, et, tm, on, T, R, L)
    counts = exact["counts"].astype(np.int64)
    t_, b_ = int(np.argmax(counts[:, 1])), 1
    bounds = counts.copy()
    bounds[:, L + 1] = 0
    bounds[t_, b_] = counts[t_, b_] // 2                                       # overflows class (t_, 1)
    n_rows = int(bounds.sum()) + 1
    got = _layout(nt, ei, et, tm, on, T, R, L, bounds=bounds, n_rows=n_rows)
    assert got["flags"][3] == 1
    assert (got["perm"][n_rows:] == CANARY).all() and (got["nt"][n_rows:] == CANARY).all()
    off = got["off"]
    ntn, dist = nt.cpu().numpy(), got["dist"]
    for k in range(T * (L + 2)):                                               # each region holds only its class
        t, b = divmod(k, L + 2)
        reg = got["perm"][off[k]:off[k + 1]]
        real = reg[reg < N]
        assert real.size == min(counts[t, b], bounds[t, b]), (t, b)
        assert (ntn[real] == t).all() and (np.minimum(dist[real], L + 1) == b).all()
        assert (got["nt"][off[k]:off[k + 1]] == t).all()
    assert (got["ei"] >= 0).all() and (got["ei"] < n_rows).all()

    m = _gnn(T, R, L).eval()
    x = torch.randn(N, 32, device=dev)
    tsig = trim.TrimSignature(bounds, L)
    with torch.no_grad():
        out = m(x, nt, tm, ei, et, out_nodes=on, trim_signature=tsig)
    assert torch.isnan(out).all()
    lay = trim.get_layout(nt, ei, et, tm, on, T, R, L, tsig, P.get_plan(nt, ei, et, tm, T, R).pairs)
    assert int(lay.flags_dev[3]) == 1
    with pytest.raises(ValueError):
        lay.check()
    bad = torch.tensor([0, N], device=dev)
    ok = trim.TrimSignature(counts + 2, L)
    with torch.no_grad():
        out = m(x, nt, tm, ei, et, out_nodes=bad, trim_signature=ok)
    assert torch.isnan(out).all()
    with pytest.raises(IndexError):
        trim.get_layout(nt, ei, et, tm, bad, T, R, L, ok, P.get_plan(nt, ei, et, tm, T, R).pairs).check()
    with pytest.raises(ValueError):
        trim.TrimSignature(counts[:, :L + 1], L)
    with pytest.raises(ValueError):
        m(x, nt, tm, ei, et, trim_signature=ok)


# ---------------------------------------------------------------------------------------------------------------------
# 5. / 6. graphed trimmed forward and training step

def _graphed_setup(B=4, L=3, seed=9):
    members, seeds, T, R = _sampled_members(B, 3, 8, seed=seed)
    plans = [P.get_plan(mb[1], mb[3], mb[4], mb[2], T, R) for mb in members]
    counts = [max(p.type_count[t] for p in plans) + 3 for t in range(T)]
    pairs = {pr for p in plans for pr in p.pairs}
    sig = graphed.GraphSignature(counts, max(p.n_edges for p in plans) + 50, pairs, R, members[0][0].shape[1])
    paper = [t for t in range(T) if int(seeds[0][0]) == plans[0].type_row0[t] and plans[0].type_count[t]][0]
    C = seeds[0].numel()
    rows = torch.arange(C, device=seeds[0].device) + int(sig.row0[paper])
    tsig = trim.TrimSignature.for_batches(members, seeds, L, 0.1, num_types=T, num_relations=R)
    return members, seeds, plans, sig, paper, rows, tsig, T, R


def test_graphed_trimmed_forward_lays_out_every_replayed_batch():
    L = 3
    members, seeds, _, sig, _, rows, tsig, T, R = _graphed_setup(L=L)
    m = _gnn(T, R, L, F_in=8).eval()
    gf = graphed.GraphedForward(lambda x, nt, tm, ei, et: m(x, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig),
                                sig, "cuda", per_node=False)
    for rep in range(2):
        for mb, s in zip(members, seeds):
            out = gf(*mb[:5])
            with torch.no_grad():
                exact = m(*mb[:5], out_nodes=s)
                full = m(*mb[:5])[s]
            assert torch.equal(out, exact), "replay %d differs from the eager trimmed rows" % rep
            assert (out - full).abs().max().item() <= FWD_MAX_ABS
    assert gf.graph is not None
    # the layout inside the graph is not reachable: an eager rebuild on the static buffers checks the last batch
    trim.get_layout(gf.nt, gf.ei, gf.et, gf.tm, rows, T, R, L, tsig, gf.plan.pairs).check()


def _graphed_steps(m, head, sig, rows, tsig, paper, trimmed, autocast):
    C = rows.numel()

    def loss_fn(x, nt, tm, ei, et, targets):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            h = m(x, nt, tm, ei, et, out_nodes=rows, trim_signature=tsig) if trimmed else m(x, nt, tm, ei, et)[rows]
            return F.nll_loss(F.log_softmax(head(h).float(), -1), targets[paper][:C], ignore_index=-100)

    params = list(m.parameters()) + list(head.parameters())
    return graphed.GraphedTrainStep(loss_fn, sig, "cuda", params=params, targets={paper: ((), torch.int64, -100)}), params


@pytest.mark.parametrize("autocast", [False, True])
def test_graphed_trimmed_train_step_matches_eager_and_untrimmed(autocast):
    L = 3
    members, seeds, plans, sig, paper, rows, tsig, T, R = _graphed_setup(L=L)
    m = _gnn(T, R, L, F_in=8, dropout=0.0).train()
    torch.manual_seed(3)
    head = torch.nn.Linear(64, 5).to(rows.device)
    st_trim, params = _graphed_steps(m, head, sig, rows, tsig, paper, True, autocast)
    st_full, _ = _graphed_steps(m, head, sig, rows, tsig, paper, False, autocast)
    bar = BF16_GRAD_REL_FRO if autocast else GRAPHED_GRAD_REL_FRO
    n_loss = 0
    g_trim = g_full = None                       # each graph writes the .grad tensors it captured, whatever p.grad is now
    with _deterministic(True):
        for rep in range(2):
            for b, mb in enumerate(members):
                y = torch.randint(0, 5, (plans[b].type_count[paper],), generator=torch.Generator().manual_seed(b))
                loss, = st_trim(*mb[:5], targets={paper: y.to(rows.device)})
                loss = loss.clone()
                g_trim = g_trim or [p.grad for p in params]
                for p in params:
                    p.grad = None
                st_trim._rebuild_plan()                                        # eager, on the same padded batch
                ref = st_trim.loss_fn(st_trim.x, st_trim.nt, st_trim.tm, st_trim.ei, st_trim.et, st_trim.y)
                ref.backward()
                ref = ref.detach()                          # a live autograd graph would break the next capture
                assert torch.equal(loss, ref), "rep %d batch %d" % (rep, b)
                n_loss += 1
                for p in params:
                    p.grad = None
                loss_f, = st_full(*mb[:5], targets={paper: y.to(rows.device)})
                g_full = g_full or [p.grad for p in params]
                torch.cuda.synchronize()
                assert _rel(loss, loss_f) <= bar
                for g, f in zip(g_trim, g_full):
                    assert torch.isfinite(g).all()
                    assert _rel(g, f) <= bar, "rel fro %.3g" % _rel(g, f)
    assert n_loss == 8
