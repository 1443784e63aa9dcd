"""The peer-memory halo exchange of the multi-GPU forward (csrc/plan.cu) on ONE GPU.

A peer table is a device int64 array of the data_ptr()s of W separate allocations on this GPU: the halo kernels only
dereference those pointers, so every kernel runs here exactly as it runs over NVLink.

Kernel tests (bitwise against torch): hgt_halo_pull_split (every VPL instance and both sides of each VPL boundary, a
tail of every rows-per-pass count RB, `order` NULL and a permutation of a subset of the rows, both publish areas, W = 1
to 4, a grid-stride case), hgt_halo_push_split (the same widths, items to several peers including self with repeated
sources, both destination areas, a grid-stride case), hgt_halo_pull (float4 and scalar rows, both areas) and
hgt_gather_rows (float4 and scalar paths).  Every output starts as a sentinel, so a write outside the addressed rows, or
an fp32 row written for a row this rank does not own, shows.  The inputs hold subnormals, values at bf16 rounding ties
(of hi and of lo) and magnitudes up to 3.4e38; no inf or NaN (inf - inf would make lo a NaN of unspecified payload).

Emulated p2p sharded forward: the ShardedGraphs of every rank of W = 2, 3, 4 live in one process and share a stand-in
symmetric-memory handle (the device table of every rank's publish buffer, a barrier with nothing to wait for: one stream
orders all ranks' work).  Every rank publishes before any rank pulls; then the real ShardedGraph.forward runs rank by
rank, for two chained layers (publish area 0, then area 1).  Each rank's output must be bitwise equal to the same layer
run on x[local_global] without an exchange, and close to the float64 oracle of the full graph on the owned rows.  The
push variant (halo_mode="push") is emulated the same way with a push plan built from every rank's pull tables.
"""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hgt_oracle                 # noqa: E402
from pyhgt_b200 import _lib, sharded, synth   # noqa: E402

SPLIT_WIDTHS = [8, 64, 72, 128, 136, 256, 264, 400, 512, 520, 1024]   # VPL 1 | 2 | 4 | 8 boundaries at 128, 256, 512
SENT_F32 = -8.5e-37                # sentinels: bit patterns no kernel under test writes for these inputs
SENT_BF16 = -3.0e-37

# float32 bit patterns put into every input
SPECIAL_BITS = [
    0x00000001, 0x80000001, 0x007FFFFF, 0x00400000, 0x0000FFFF,   # subnormals
    0x00008000, 0x00018000,                                       # subnormal hi ties (even, odd)
    0x3F808000, 0x3F818000, 0xBF808000, 0xC2FE8000,               # hi ties: round down to even, up to even
    0x3F800101, 0x3F800301, 0xBF800101,                           # lo ties (9 significant bits left for lo)
    0x7F000000, 0x7F7F0000, 0x7F7F7FFF, 0xFF7F7FFF, 0xFE912345,   # large magnitudes (0x7F7F7FFF: largest below the
    0x80000000, 0x00000000,                                       # bf16 overflow), signed zeros
]


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _rows(n, d, seed):
    """[n, d] fp32 rows on the GPU: a wide spread of magnitudes with SPECIAL_BITS at random places."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g) * torch.exp2(torch.randint(-30, 30, (n, d), generator=g).float())
    flat = x.view(-1).view(torch.int32)
    sp = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in SPECIAL_BITS], dtype=torch.int32)
    k = min(flat.numel(), 4 * sp.numel())
    flat[torch.randperm(flat.numel(), generator=g)[:k]] = sp.repeat(4)[:k]
    return x.to(_dev())


def _split(v):
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def _same(a, b, what):
    """Bitwise equality (so -0.0 vs 0.0 and sentinel bits count)."""
    it = torch.int32 if a.dtype == torch.float32 else torch.int16
    ai, bi = a.contiguous().view(it), b.contiguous().view(it)
    bad = (ai != bi).nonzero()
    assert bad.numel() == 0, "%s: %d elements differ, first at %s" % (what, bad.shape[0], bad[0].tolist())


def _table(bufs):
    return torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=_dev())


def _i32(t):
    return t.to(torch.int32).to(_dev())


# ---- hgt_halo_pull_split ----------------------------------------------------------------------------------------------
def _pull_split_case(width, W, n_rows, use_order, slot, self_rank, seed, m=40):
    """One call: n_rows rows of a pull plan over W ranks with `m` rows per publish area.  With use_order the call
    processes a permutation of a strict subset of a larger plan, so exactly the listed rows must be written."""
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    n_plan = n_rows + (5 if use_order else 0)
    src_rank = torch.randint(0, W, (n_plan,), generator=g)
    src_row = torch.randint(0, m, (n_plan,), generator=g)
    bufs = [_rows(2 * m, width, seed * 10 + w) for w in range(W)]
    order = torch.randperm(n_plan, generator=g)[:n_rows] if use_order else None
    rows = order if use_order else torch.arange(n_rows)
    # one sentinel row before and after the n_plan addressed rows
    out = torch.full((n_plan + 2, width), SENT_F32, device=dev)
    hi = torch.full((n_plan + 2, width), SENT_BF16, dtype=torch.bfloat16, device=dev)
    lo = hi.clone()
    # every device argument is held in a local until the kernel has run: a temporary's block would go back to the
    # caching allocator at once and could hold the next argument by launch time
    tab, d_rank, d_row = _table(bufs), _i32(src_rank), _i32(src_row)
    d_order = None if order is None else _i32(order)
    _lib.call("hgt_halo_pull_split", tab.data_ptr(), d_rank.data_ptr(), d_row.data_ptr(), _lib.ptr(d_order), n_rows,
              width, self_rank, slot * m, out[1:].data_ptr(), hi[1:].data_ptr(), lo[1:].data_ptr(), _stream())
    allb = torch.stack(bufs)
    sr, rw = src_rank[rows].to(dev), (slot * m + src_row[rows]).to(dev)
    v = allb[sr, rw]
    e_out, e_hi, e_lo = torch.full_like(out, SENT_F32), torch.full_like(hi, SENT_BF16), torch.full_like(lo, SENT_BF16)
    at = (rows + 1).to(dev)
    e_out[at] = torch.where((sr == self_rank)[:, None], v, torch.full_like(v, SENT_F32))
    e_hi[at], e_lo[at] = _split(v)
    what = "width %d W %d rows %d order %s slot %d self %d" % (width, W, n_rows, use_order, slot, self_rank)
    _same(out, e_out, "pull_split out_f32 " + what)
    _same(hi, e_hi, "pull_split hi " + what)
    _same(lo, e_lo, "pull_split lo " + what)


# (W, n_rows, order, slot): n_rows leaves a tail of 1, 2 and 3 rows for RB = 4 and of 1 row for RB = 2
PULL_SPLIT_PLANS = [(1, 1, False, 0), (2, 6, True, 1), (3, 7, False, 1), (4, 37, True, 0), (4, 130, False, 1),
                    (3, 131, True, 1)]


@pytest.mark.parametrize("width", SPLIT_WIDTHS)
def test_halo_pull_split_matches_torch_bitwise(width):
    for i, (W, n, use_order, slot) in enumerate(PULL_SPLIT_PLANS):
        _pull_split_case(width, W, n, use_order, slot, self_rank=i % W, seed=100 + i)


@pytest.mark.parametrize("width,rb", [(64, 4), (512, 2), (1024, 1)])
def test_halo_pull_split_grid_stride(width, rb):
    """More rows than the capped grid (16 blocks of 8 warps per SM, RB rows per warp) covers in one pass: the grid-stride
    loop turns twice and ends on a tail."""
    sm = torch.cuda.get_device_properties(_dev()).multi_processor_count
    n = 2 * sm * 16 * 8 * rb + 3
    _pull_split_case(width, 3, n, True, 1, self_rank=2, seed=7, m=300)


def test_halo_pull_split_rejects_unsupported_widths():
    dev = _dev()
    z = torch.zeros(64, dtype=torch.int32, device=dev)
    buf = torch.zeros((4, 1032), device=dev)
    tab = _table([buf])
    o = torch.empty((4, 1032), device=dev)
    h = torch.empty((4, 1032), dtype=torch.bfloat16, device=dev)
    for width in (12, 1032):
        with pytest.raises(_lib.HgtError, match="hgt_halo_pull_split"):
            _lib.call("hgt_halo_pull_split", tab.data_ptr(), z.data_ptr(), z.data_ptr(), None, 1, width, 0, 0,
                      o.data_ptr(), h.data_ptr(), h.data_ptr(), _stream())
    torch.cuda.synchronize()


# ---- hgt_halo_push_split ----------------------------------------------------------------------------------------------
def _push_case(width, W, n_items, row_base_slot, self_rank, seed, n_own=50):
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    peer = torch.randint(0, W, (n_items,), generator=g)
    peer[:W] = torch.arange(W)                                   # every peer, self included, gets items
    src = torch.randint(0, n_own, (n_items,), generator=g)       # repeated sources
    cnt = torch.bincount(peer, minlength=W)
    max_local = int(cnt.max()) + 3
    dst = torch.empty(n_items, dtype=torch.int64)
    for p in range(W):                                           # distinct destination rows inside every peer
        sel = (peer == p).nonzero().flatten()
        dst[sel] = torch.randperm(max_local, generator=g)[:sel.numel()]
    x_own = _rows(n_own, width, seed)
    row_base = row_base_slot * max_local
    his = [torch.full((2 * max_local + 2, width), SENT_BF16, dtype=torch.bfloat16, device=dev) for _ in range(W)]
    los = [h.clone() for h in his]
    xl = torch.full((max_local + 2, width), SENT_F32, device=dev)
    d_peer, d_src, d_dst = _i32(peer), _i32(src), _i32(dst)
    t_hi, t_lo = _table([h[1:] for h in his]), _table([l_[1:] for l_ in los])
    _lib.call("hgt_halo_push_split", x_own.data_ptr(), d_peer.data_ptr(), d_src.data_ptr(), d_dst.data_ptr(), n_items,
              width, self_rank, row_base, t_hi.data_ptr(), t_lo.data_ptr(), xl[1:].data_ptr(), _stream())
    what = "width %d W %d items %d slot %d self %d" % (width, W, n_items, row_base_slot, self_rank)
    for p in range(W):
        sel = (peer == p).nonzero().flatten()
        v = x_own[src[sel].to(dev)]
        e_hi = torch.full_like(his[p], SENT_BF16)
        e_lo = e_hi.clone()
        at = (1 + row_base + dst[sel]).to(dev)
        e_hi[at], e_lo[at] = _split(v)
        _same(his[p], e_hi, "push hi of peer %d, %s" % (p, what))
        _same(los[p], e_lo, "push lo of peer %d, %s" % (p, what))
        if p == self_rank:
            e_xl = torch.full_like(xl, SENT_F32)
            e_xl[(1 + dst[sel]).to(dev)] = v
            _same(xl, e_xl, "push fp32 rows, " + what)


@pytest.mark.parametrize("width", SPLIT_WIDTHS)
def test_halo_push_split_matches_torch_bitwise(width):
    for i, (W, n, slot) in enumerate([(1, 3, 0), (2, 9, 1), (3, 40, 0), (4, 77, 1)]):
        _push_case(width, W, n, slot, self_rank=(i + 1) % W, seed=200 + i)


@pytest.mark.parametrize("width", [64, 1024])
def test_halo_push_split_grid_stride(width):
    """More items than the capped grid (8 blocks of 8 warps per SM, one item per warp) covers in one pass."""
    sm = torch.cuda.get_device_properties(_dev()).multi_processor_count
    _push_case(width, 4, 2 * sm * 8 * 8 + 5, 1, self_rank=1, seed=9)


# ---- hgt_halo_pull ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [4, 12, 100, 1024, 78, 30])
@pytest.mark.parametrize("slot", [0, 1])
def test_halo_pull_matches_torch_bitwise(width, slot):
    """float4 rows (width % 4 == 0) and float-by-float rows (width 78, 30, or an output that is not 16-byte aligned)."""
    dev = _dev()
    g = torch.Generator().manual_seed(width * 2 + slot)
    W, m, n = 3, 30, 75
    src_rank, src_row = torch.randint(0, W, (n,), generator=g), torch.randint(0, m, (n,), generator=g)
    bufs = [_rows(2 * m, width, 300 + w) for w in range(W)]
    want = torch.stack(bufs)[src_rank.to(dev), (slot * m + src_row).to(dev)]
    tab, d_rank, d_row = _table(bufs), _i32(src_rank), _i32(src_row)
    for shift in ((1, 0) if width % 4 == 0 else (0,)):           # shift 1: the output starts one float past 16 bytes
        flat = torch.full(((n + 2) * width + 1,), SENT_F32, device=dev)
        out = flat[width + shift:width + shift + n * width]
        _lib.call("hgt_halo_pull", tab.data_ptr(), d_rank.data_ptr(), d_row.data_ptr(), n, width, slot * m,
                  out.data_ptr(), _stream())
        exp = torch.full_like(flat, SENT_F32)
        exp[width + shift:width + shift + n * width] = want.reshape(-1)
        _same(flat, exp, "halo_pull width %d slot %d shift %d" % (width, slot, shift))


# ---- hgt_gather_rows --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width,in_shift,out_shift", [(64, 0, 0), (30, 0, 0), (64, 1, 0), (64, 0, 1), (1024, 0, 0)])
def test_gather_rows_matches_index_select(width, in_shift, out_shift):
    """float4 path (aligned, width % 4 == 0) and the scalar path: width 30, input or output one float off 16 bytes."""
    dev = _dev()
    g = torch.Generator().manual_seed(width + 7 * in_shift + 13 * out_shift)
    n_in, n = 90, 200
    perm = torch.randint(0, n_in, (n,), generator=g)             # repeats
    src = _rows(n_in, width, 400).reshape(-1)
    inb = torch.empty(n_in * width + 1, device=dev)
    inb[in_shift:in_shift + n_in * width] = src
    outb = torch.full(((n + 1) * width + 1,), SENT_F32, device=dev)
    d_perm = _i32(perm)
    _lib.call("hgt_gather_rows", inb[in_shift:].data_ptr(), d_perm.data_ptr(), n, width, outb[out_shift:].data_ptr(),
              _stream())
    exp = torch.full_like(outb, SENT_F32)
    exp[out_shift:out_shift + n * width] = src.view(n_in, width)[perm.to(dev)].reshape(-1)
    _same(outb, exp, "gather_rows width %d in+%d out+%d" % (width, in_shift, out_shift))


# ---- emulated p2p sharded forward -------------------------------------------------------------------------------------
class _Handle:
    """Stand-in for a symmetric-memory handle: the device table of every rank's buffer, and a barrier with nothing to
    wait for (one stream orders every rank's work)."""

    def __init__(self, bufs):
        self.table = _table(bufs)
        self.buffer_ptrs_dev = self.table.data_ptr()

    def barrier(self, channel=0):
        pass


# name: (d, H, T, R, use_norm, use_RTE, linear_impl)
CASES = {
    "d64_rte_norm": (64, 4, 3, 4, True, True, 0),
    "d256_t4r4": (256, 8, 4, 4, True, False, 0),
    "d400_rte": (400, 8, 3, 3, True, True, 0),
    "d512": (512, 8, 3, 3, False, False, 0),
    "d48_pull": (48, 4, 3, 4, True, True, 0),         # width not split-able: hgt_halo_pull, the layer splits x itself
    "d78_scalar": (78, 3, 3, 4, True, True, 0),       # width % 4 != 0: hgt_halo_pull's scalar rows
    "d64_simt": (64, 4, 3, 4, True, True, 1),         # linear_impl 1: no split, fp32 pull
}
MODES = ["fp32", "autocast_bf16", "matmul_medium"]
# Worst max|out - float64| / max(1, max|ref|) over both layers, all cases and W = 2, 3, 4, measured on an H100 80GB HBM3
# (700 W power limit): fp32 4.1e-6 (d400_rte), bf16 autocast 1.3e-3 (d64_rte_norm), matmul precision "medium" 2.1e-3
# (d400_rte).  Each bound is about 10x that.
ERR_BOUND = {"fp32": 4e-5, "autocast_bf16": 1.3e-2, "matmul_medium": 2e-2}
ERR_REPORT = os.environ.get("HGT_HALO_ERR_REPORT")   # optional JSON file collecting the measured errors

_cache = {}


def _graph(T, R, seed):
    """Isolated destinations, self loops, duplicate edges, a few nodes of the out-of-range type T, and type T - 1 with
    only 2 nodes, so that for W > 2 some rank owns none of it."""
    g = synth.make_random(400, 2000, T, R, seed=seed, isolated_frac=0.15, self_loops=30, duplicate_edges=40)
    nt = g.node_type.clone()
    gen = torch.Generator().manual_seed(seed + 1)
    few = (nt == T - 1).nonzero().flatten()
    nt[few[2:]] = torch.randint(0, T - 1, (few.numel() - 2,), generator=gen)
    zero = (nt == 0).nonzero().flatten()
    nt[zero[torch.randperm(zero.numel(), generator=gen)[:6]]] = T
    g.node_type = nt
    return g


def _case(name):
    """Graph, two layers, their float64 oracle outputs (layer 2 on the float64 layer-1 output) and the input."""
    if name not in _cache:
        import pyhgt_b200
        d, H, T, R, norm, rte, impl = CASES[name]
        dev = _dev()
        g = _graph(T, R, seed=list(CASES).index(name) + 31)
        torch.manual_seed(d + H)
        convs = [pyhgt_b200.HGTConv(d, d, T, R, H, 0.2, norm, rte).to(dev).eval() for _ in range(2)]
        for c in convs:
            c.linear_impl = impl
        x = torch.randn(g.num_nodes, d, generator=torch.Generator().manual_seed(d))
        kw = dict(num_types=T, num_relations=R, n_heads=H, use_norm=norm, use_RTE=rte)
        refs, h = [], x.double()
        for c in convs:
            p = {k: v.detach().double().cpu() for k, v in c.state_dict().items()}
            h = hgt_oracle.hgt_forward_ref_port(p, h, g.node_type, g.edge_index, g.edge_type, g.edge_time, **kw)[0]
            refs.append(h)
        _cache[name] = dict(g=g, convs=convs, x=x.to(dev), refs=refs, shards={})
    return _cache[name]


def _shards(c, W, d):
    """Every rank's ShardedGraph of W, halo_mode "p2p", sharing a stand-in handle over one [2 * max_owned, d] publish
    buffer per rank."""
    if W not in c["shards"]:
        g, dev = c["g"], _dev()
        shs = [sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, g.num_types,
                                          g.num_relations, r, W, dev, halo_mode="p2p") for r in range(W)]
        m = max(shs[0].max_owned, 1)
        bufs = [torch.full((2 * m, d), float("nan"), device=dev) for _ in range(W)]
        hdl = _Handle(bufs)
        for sh, b in zip(shs, bufs):
            sh._symm = (b, hdl)
        assert W <= 2 or any(sh.active_per_type[g.num_types - 1] == 0 for sh in shs)
        c["shards"][W] = shs
    return c["shards"][W]


def _direct(conv, sh, x_local, out_map):
    """The same layer on the rows the exchange should deliver, without an exchange."""
    out, _, _ = conv._forward_impl(x_local, sh.node_type, sh.edge_index, sh.edge_type,
                                   sh.edge_time if conv.use_RTE else None, want_att=False, save=False,
                                   active_per_type=sh.active_per_type, out_map=out_map, out_rows=sh.n_owned,
                                   kv_runs=sh.kv_runs)
    return out


def _out_map(sh):
    om = torch.full((sh.n_owned + sh.n_halo,), -1, dtype=torch.int32, device=_dev())
    om[sh.own_rows] = torch.arange(sh.n_owned, dtype=torch.int32, device=_dev())
    return om


def _pull_layer(shs, conv, xg, slot, plain_rank=None):
    """Publish every rank's rows (in place through input_buffer, or, for plain_rank, as a plain tensor that forward
    copies into its publish area), then run each rank's ShardedGraph.forward.  The plain rank runs first: its copy is
    the only publish that happens inside a forward."""
    d, dev = xg.shape[1], xg.device
    pubs = []
    for r, sh in enumerate(shs):
        own = xg[sh.owned_global.to(dev)]
        if r == plain_rank:
            assert sh._slot == slot
            pubs.append(own.clone())
        else:
            p = sh.input_buffer(d, slot)
            p.copy_(own)
            pubs.append(p)
    outs = [None] * len(shs)
    for r in sorted(range(len(shs)), key=lambda r: r != plain_rank):
        with torch.no_grad():
            outs[r] = shs[r].forward(conv, pubs[r])
        assert shs[r]._slot == slot ^ 1
    return outs


class _Mode:
    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.prec = torch.get_float32_matmul_precision()
        self.ac = None
        if self.mode == "matmul_medium":
            torch.set_float32_matmul_precision("medium")
        elif self.mode == "autocast_bf16":
            self.ac = torch.autocast("cuda", dtype=torch.bfloat16)
            self.ac.__enter__()

    def __exit__(self, *exc):
        if self.ac is not None:
            self.ac.__exit__(*exc)
        torch.set_float32_matmul_precision(self.prec)


def _record(key, err):
    if ERR_REPORT:
        data = json.load(open(ERR_REPORT)) if os.path.exists(ERR_REPORT) else {}
        data[key] = err
        with open(ERR_REPORT, "w") as f:
            json.dump(data, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_p2p_forward_matches_direct_and_float64(name, mode):
    c = _case(name)
    d = CASES[name][0]
    dev = _dev()
    n = c["g"].num_nodes
    worst = 0.0
    for W in (2, 3, 4):
        shs = _shards(c, W, d)
        xg = c["x"]
        with _Mode(mode):
            for layer, conv in enumerate(c["convs"]):
                outs = _pull_layer(shs, conv, xg, slot=layer, plain_rank=0 if layer == 0 else None)
                nxt = torch.full((n, d), float("nan"), device=dev)
                for r, sh in enumerate(shs):
                    with torch.no_grad():
                        ref = _direct(conv, sh, xg[sh.local_global.to(dev)], sh._out_map)
                    _same(outs[r], ref, "%s %s W %d layer %d rank %d: p2p forward vs direct" % (name, mode, W, layer, r))
                    nxt[sh.owned_global.to(dev)] = outs[r]
                ref64 = c["refs"][layer]
                err = ((nxt.double().cpu() - ref64).abs().max() / ref64.abs().max().clamp_min(1.0)).item()
                worst = max(worst, err)
                xg = nxt
    _record("%s/%s" % (name, mode), worst)
    assert worst <= ERR_BOUND[mode], "%s %s: error vs float64 %.3g > %.3g" % (name, mode, worst, ERR_BOUND[mode])


# ---- emulated push ----------------------------------------------------------------------------------------------------
def _push_plans(shs, d):
    """Every rank's `_push` state from all ranks' pull tables: owner o gets (peer c, src pull_row_c[j], dst j) for every
    local row j of every rank c with pull_rank_c[j] == o; hi / lo buffers of 2 * max_local rows per rank."""
    dev = _dev()
    W = len(shs)
    max_local = max(sh.n_owned + sh.n_halo for sh in shs)
    his = [torch.full((2 * max_local, d), float("nan"), dtype=torch.bfloat16, device=dev) for _ in range(W)]
    los = [h.clone() for h in his]
    h_hi, h_lo = _Handle(his), _Handle(los)
    for o, sh in enumerate(shs):
        peer, src, dst = [], [], []
        for cr, shc in enumerate(shs):
            j = (shc.pull_rank == o).nonzero().flatten()
            peer.append(torch.full_like(j, cr))
            src.append(shc.pull_row[j].long())
            dst.append(j)
        sh._push = dict(d=d, peer=_i32(torch.cat(peer)), src=_i32(torch.cat(src)), dst=_i32(torch.cat(dst)),
                        hi=his[o], lo=los[o], h_hi=h_hi, h_lo=h_lo, max_local=max_local, slot=0)
        sh.halo_mode = "push"


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("name", ["d64_rte_norm", "d256_t4r4"])
def test_emulated_push_matches_pull(name, W):
    c = _case(name)
    d = CASES[name][0]
    dev = _dev()
    g = c["g"]
    built = [sharded.ShardedGraph.build(g.node_type, g.edge_index, g.edge_type, g.edge_time, g.num_types,
                                        g.num_relations, r, W, dev, halo_mode="push") for r in range(W)]
    _push_plans(built, d)
    pull_shs = _shards(c, W, d)
    for rnd, conv in enumerate(c["convs"]):
        xg = _rows(g.num_nodes, d, 500 + rnd).clamp(-1e3, 1e3) if rnd else c["x"]
        got = [sh.exchange(xg[sh.owned_global.to(dev)], split=True) for sh in built]   # every owner pushes first
        want = _pull_layer(pull_shs, conv, xg, slot=rnd)
        for r, sh in enumerate(built):
            assert sh._push["slot"] == (rnd + 1) % 2
            x_local, (hi, lo) = got[r]
            e_hi, e_lo = _split(xg[sh.local_global.to(dev)])
            _same(hi, e_hi, "%s W %d round %d rank %d: pushed hi" % (name, W, rnd, r))
            _same(lo, e_lo, "%s W %d round %d rank %d: pushed lo" % (name, W, rnd, r))
            _same(x_local[sh.own_rows], xg[sh.owned_global.to(dev)], "%s W %d rank %d: owned fp32 rows" % (name, W, r))
            with torch.no_grad():
                out, _, _ = conv._forward_impl(x_local, sh.node_type, sh.edge_index, sh.edge_type,
                                               sh.edge_time if conv.use_RTE else None, want_att=False, save=False,
                                               active_per_type=sh.active_per_type, out_map=_out_map(sh),
                                               out_rows=sh.n_owned, x_split=(hi, lo), kv_runs=sh.kv_runs)
            _same(out, want[r], "%s W %d round %d rank %d: push forward vs pull forward" % (name, W, rnd, r))
