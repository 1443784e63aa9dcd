"""The host bounds of sync-free plans really bound what the tile planner emits, and the poison the GPU tests put past the
device counts stays in range (no GPU needed).

Sync-free plans (plan.build_plan(..., host_meta=...)), every SourceIndex and the trimmed range views size their tile and
hub arrays with plan.tile_bounds and keep those sizes as the host-side n_tiles / n_split / n_hubs.  hgt_plan_tiles
(csrc/plan.cu, k_tile_emit_counts / k_tile_write) drops tiles and hubs past the arrays silently, so a bound that is too
small would lose work without an error.  `emit` restates the planner in numpy; the tests run it over degree sequences
built to push each term of the bound.

tests/test_gpu_sync_free_instances.py fills the slots past the device counts with poison_tails; here it runs on CPU
tensors: every entry it writes is in range (so a kernel that read to the bound computes wrong numbers, never out of
bounds), and a numpy consumer that reads to the bound instead of the count gets a different agg / dq.
"""
import numpy as np
import pytest
import torch

from pyhgt_b200 import plan as P
from tests.test_gpu_sync_free_instances import poison_tails


def emit(row_ptr, target, split, ranges=None):
    """numpy restatement of hgt_plan_tiles / hgt_plan_range_tiles: the tiles [dst, dst_end or -(slot+1), e0, e1] and
    hubs [dst, first slot, pieces, 0] over the rows of row_ptr (or the ascending, disjoint row ranges).  A row starts a
    tile if it opens its range, follows a hub, or its cost prefix 2 * row_ptr[k] + k enters a new bucket of 2 * target
    units; a hub (deg > split) takes ceil(deg / split) pieces of its own."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    n = rp.size - 1
    ranges = [(0, n)] if ranges is None else [(a, b) for a, b in ranges if b > a]
    tc = 2 * target
    tiles, hubs, slot = [], [], 0
    for a, b in ranges:
        for k in range(a, b):
            deg = int(rp[k + 1] - rp[k])
            if deg > split:
                pieces = -(-deg // split)
                per = -(-deg // pieces)
                hubs.append([k, slot, pieces, 0])
                for i in range(pieces):
                    e0 = int(rp[k]) + i * per
                    tiles.append([k, -(slot + i) - 1, e0, min(int(rp[k + 1]), e0 + per)])
                slot += pieces
                continue
            if k == a or rp[k] - rp[k - 1] > split or (2 * rp[k] + k) // tc != (2 * rp[k - 1] + k - 1) // tc:
                tiles.append([k, -1, int(rp[k]), -1])
    # close the whole-row tiles (k_tile_close): up to the next tile's row or the end of the range
    ends = {a: b for a, b in ranges}
    starts = sorted(ends)
    for i, t in enumerate(tiles):
        if t[1] == -1 and t[3] == -1:
            r_end = ends[starts[np.searchsorted(starts, t[0], side="right") - 1]]
            nxt = tiles[i + 1][0] if i + 1 < len(tiles) else n
            t[1] = min(nxt, r_end)
            t[3] = int(rp[t[1]])
    return tiles, hubs, slot


def _rp(deg):
    return np.concatenate([[0], np.cumsum(np.asarray(deg, dtype=np.int64))])


def _check(deg, ranges=None, n_rows=None):
    """The planner's counts over `deg` within plan.tile_bounds as build_plan / source_index (or trim._range_view)
    compute them; n_rows: the rows the bound counts (a source index: kv rows; default all)."""
    rp = _rp(deg)
    n = rp.size - 1
    E = int(rp[-1])
    tiles, hubs, n_split = emit(rp, P.TILE_TARGET_EDGES, P.TILE_SPLIT_EDGES, ranges)
    max_tiles, max_split, max_hubs = P.tile_bounds(n if n_rows is None else n_rows, E, 0 if ranges is None else
                                                   len(ranges))
    assert len(tiles) <= max_tiles, (len(tiles), max_tiles)
    assert len(hubs) <= max_hubs, (len(hubs), max_hubs)
    assert n_split <= max_split, (n_split, max_split)
    assert (max_split > 0) == (E > P.TILE_SPLIT_EDGES)
    return tiles, hubs, n_split


S = P.TILE_SPLIT_EDGES
TGT = P.TILE_TARGET_EDGES


def _bucket_edges(n):
    """Degrees that put every destination on a cost-bucket boundary: rows alternate costs 2 * TILE_TARGET_EDGES + 1 and
    2 * TILE_TARGET_EDGES - 1, so every row's cost prefix enters a new bucket and every row starts a tile."""
    return [TGT if i % 2 == 0 else TGT - 1 for i in range(n)]


SEQUENCES = {
    "hubs_at_split_plus_one": [S + 1] * 200,
    "hubs_at_split_plus_one_with_rows_between": [S + 1, 0, 3] * 150,
    "hubs_at_multiples_of_split": [S * m for m in range(1, 40)] + [2 * S] * 50,
    "hubs_at_multiples_plus_one": [S * m + 1 for m in range(1, 40)],
    "every_row_on_a_bucket_boundary": _bucket_edges(5000),
    "every_row_its_own_bucket": [TGT] * 4000,
    "boundaries_and_hubs": (_bucket_edges(7) + [S + 1]) * 300,
    "long_zero_runs": ([0] * 5000 + [1]) * 30 + [0] * 20000,
    "zero_runs_between_hubs": ([0] * 3000 + [S + 1]) * 40,
    "E_just_below_split": [1] * S,
    "E_at_split_one_row": [S],
    "E_just_above_split_no_hub": [1] * (S + 1),
    "E_just_above_split_one_hub": [S + 1],
    "E_just_above_split_two_rows": [S, 1],
    "nodes_without_edges": [0] * 10000,
    "one_row": [0],
    "one_hub_holds_every_edge": [0] * 500 + [100 * S + 7] + [0] * 500,
    "one_hub_holds_every_edge_first": [37 * S - 1] + [0] * 2000,
    "one_hub_holds_every_edge_last": [0] * 2000 + [5 * S + 1],
    "mixed_random": list(np.random.default_rng(0).zipf(1.6, 20000).clip(0, 20 * S) - 1),
}


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_bounds_hold_for_whole_plans(name):
    _check(SEQUENCES[name])


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_bounds_hold_for_source_indices(name):
    """A SourceIndex counts its bound over the owned rows (kv_rows or P * 240) and all E entries, while the trailing
    no-work row's entries get no tile: the same degree sequence with a tail of entries past ptr[n_rows]."""
    deg = list(SEQUENCES[name])
    tiles, hubs, n_split = emit(_rp(deg), TGT, S)
    E_total = sum(deg) + 3 * S                                # entries of the trailing row: counted in E, no tiles
    max_tiles, max_split, max_hubs = P.tile_bounds(len(deg), E_total)
    assert len(tiles) <= max_tiles and len(hubs) <= max_hubs and n_split <= max_split


@pytest.mark.parametrize("name", list(SEQUENCES))
def test_bounds_hold_for_range_tiles(name):
    """Trimmed views (trim._range_view): tiles over row ranges, each range opening a tile of its own."""
    deg = SEQUENCES[name]
    n = len(deg)
    rng = np.random.default_rng(len(name))
    cuts = np.unique(np.concatenate([[0, n], rng.integers(0, n + 1, 2 * min(n, 60))]))
    ranges = [(int(a), int(b)) for a, b in zip(cuts[:-1:2], cuts[1::2])]
    _check(deg, ranges=ranges)
    _check(deg, ranges=[(k, k + 1) for k in range(0, n, 2)][:500])      # many one-row ranges


def test_restatement_closes_tiles_like_the_planner():
    """emit's tiles cover every row of the ranges exactly once, and hub pieces cover their row's edges."""
    deg = SEQUENCES["boundaries_and_hubs"][:200] + [0, 0, 5]
    rp = _rp(deg)
    for ranges in (None, [(0, 17), (30, 31), (40, 203)]):
        tiles, hubs, _ = emit(rp, TGT, S, ranges)
        seen = []
        for t in tiles:
            if t[1] < 0:
                if t[2] == rp[t[0]]:
                    seen.append(t[0])                         # the first piece of a hub
                assert rp[t[0]] <= t[2] < t[3] <= rp[t[0] + 1]
            else:
                seen.extend(range(t[0], t[1]))
                assert t[2] == rp[t[0]] and t[3] == rp[t[1]]
        want = list(range(len(deg))) if ranges is None else [k for a, b in ranges for k in range(a, b)]
        assert seen == want


# ---------------------------------------------------------------------------------------------------------------------
# the poison of the GPU tests

def _graph_tiles(deg, split):
    """(row_ptr, tiles, hubs, counts, bounds) of a small graph with split threshold `split`, arrays sized as a sync-free
    plan sizes them."""
    rp = _rp(deg)
    tiles, hubs, n_split = emit(rp, 4, split)
    b_t, b_s, b_h = P.tile_bounds(len(deg), int(rp[-1]))
    t = torch.zeros((b_t, 4), dtype=torch.int32)
    h = torch.zeros((max(b_h, 1), 4), dtype=torch.int32)
    if tiles:
        t[:len(tiles)] = torch.tensor(tiles, dtype=torch.int32)
    if hubs:
        h[:len(hubs)] = torch.tensor(hubs, dtype=torch.int32)
    counts = (len(tiles), n_split, len(hubs))
    bounds = (b_t if len(deg) else 0, b_s, b_h if b_s else 0)
    return torch.from_numpy(rp), t, h, counts, bounds


GRAPHS = {
    "hubs": [3, 0, 40, 7, 1, 0, 0, 17, 2, 25, 5] * 6,
    "no_hub_above_split": [3, 1, 0, 2, 4] * 20,
    "one_hub": [0] * 30 + [97] + [0] * 30,
    "no_edges": [0] * 50,
}


@pytest.fixture
def small_split(monkeypatch):
    monkeypatch.setattr(P, "TILE_SPLIT_EDGES", 8)
    monkeypatch.setattr(P, "TILE_TARGET_EDGES", 4)
    return 8


@pytest.mark.parametrize("name", list(GRAPHS))
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_poison_stays_in_range(name, seed, small_split):
    deg = GRAPHS[name]
    rp, tiles, hubs, counts, bounds = _graph_tiles(deg, small_split)
    n, E = len(deg), int(rp[-1])
    real_t, real_h = tiles.clone(), hubs.clone()
    t_rows, h_rows = poison_tails(tiles, hubs, counts, bounds, rp, seed)
    assert len(t_rows) == bounds[0] - counts[0] and len(h_rows) == max(bounds[2] - counts[2], 0)
    assert torch.equal(tiles[:counts[0]], real_t[:counts[0]]) and torch.equal(hubs[:counts[2]], real_h[:counts[2]])
    for dst, y, e0, e1 in tiles[counts[0]:bounds[0]].tolist():
        assert 0 <= dst < n and 0 <= e0 <= E
        if y < 0:
            assert -y - 1 < bounds[1] and e0 <= e1 <= E            # a hub piece: slot below the n_split bound
        else:
            assert dst < y <= n and e0 <= rp[y]                     # whole rows [dst, y) from edge e0 to row_ptr[y]
    for dst, s0, k, z in hubs[counts[2]:bounds[2]].tolist():
        assert 0 <= dst < n and k >= 1 and 0 <= s0 and s0 + k <= bounds[1] and z == 0
    if name == "hubs":
        assert bounds[1] > counts[1] and bounds[0] - counts[0] >= 3 and bounds[2] - counts[2] >= 3


def _consume(rp, kv_row, q, k, v, tiles, hubs, n_tiles, n_hubs, n_slots):
    """One head of the edge forward and the atomic dq of the backward (dagg = 1) as the kernels walk a plan: tiles in
    order (whole rows write agg; hub pieces write a partial slot (m, l, acc)), then the hub merge.  Reads n_tiles tiles
    and n_hubs hubs, whatever the real counts are; float64."""
    n = rp.size - 1
    agg = np.zeros(n)
    dq = np.zeros(n)
    part = np.full((n_slots, 3), np.nan)

    def walk(dst, e0, e1):
        s = q[dst] * k[kv_row[e0:e1]]
        if e1 == e0:
            return -np.inf, 0.0, 0.0, s
        m = s.max()
        p = np.exp(s - m)
        return m, p.sum(), (p * v[kv_row[e0:e1]]).sum(), s

    for t in tiles[:n_tiles]:
        dst, y, e0, e1 = (int(x) for x in t)
        if y < 0:
            part[-y - 1] = walk(dst, e0, e1)[:3]
            dq[dst] += walk(dst, e0, e1)[2]
            continue
        for r in range(dst, y):
            hi = int(rp[r + 1])
            m, l, acc, _ = walk(r, e0, hi)
            agg[r] = acc / (l + 1e-16)
            dq[r] += acc
            e0 = hi
    for h in hubs[:n_hubs]:
        dst, s0, pieces = (int(x) for x in h[:3])
        w = part[s0:s0 + pieces]
        M = w[:, 0].max()
        agg[dst] = (w[:, 2] * np.exp(w[:, 0] - M)).sum() / ((w[:, 1] * np.exp(w[:, 0] - M)).sum() + 1e-16)
    return agg, dq


@pytest.mark.parametrize("name", ["hubs", "one_hub", "no_hub_above_split"])
def test_reading_to_the_bound_changes_the_result(name, small_split):
    """On the poisoned arrays, a consumer that reads to the host bounds instead of the device counts gets another agg
    or dq; reading to the counts gives the poison-free result."""
    deg = GRAPHS[name]
    rp, tiles, hubs, counts, bounds = _graph_tiles(deg, small_split)
    rng = np.random.default_rng(3)
    E = int(rp[-1])
    kv_row = rng.integers(0, 40, E)
    q, k, v = rng.normal(size=len(deg)), rng.normal(size=40), rng.normal(size=40)
    clean = _consume(rp.numpy(), kv_row, q, k, v, tiles.numpy(), hubs.numpy(), counts[0], counts[2], bounds[1])
    poison_tails(tiles, hubs, counts, bounds, rp, 0)
    t, h = tiles.numpy(), hubs.numpy()
    good = _consume(rp.numpy(), kv_row, q, k, v, t, h, counts[0], counts[2], bounds[1])
    assert all(np.array_equal(a, b) for a, b in zip(good, clean))
    # direct float64 softmax: the count-bounded walk is right
    dst = np.repeat(np.arange(len(deg)), np.diff(rp.numpy()))
    s = q[dst] * k[kv_row]
    m = np.full(len(deg), -np.inf)
    np.maximum.at(m, dst, s)
    p = np.exp(s - m[dst])
    want = np.bincount(dst, p * v[kv_row], len(deg)) / (np.bincount(dst, p, len(deg)) + 1e-16)
    np.testing.assert_allclose(good[0], want, rtol=1e-12, atol=1e-12)
    over_tiles = _consume(rp.numpy(), kv_row, q, k, v, t, h, bounds[0], counts[2], bounds[1])
    assert not all(np.array_equal(a, b, equal_nan=True) for a, b in zip(over_tiles, clean))
    if bounds[2] > counts[2]:
        over_hubs = _consume(rp.numpy(), kv_row, q, k, v, t, h, counts[0], bounds[2], bounds[1])
        assert not np.array_equal(over_hubs[0], clean[0], equal_nan=True)
