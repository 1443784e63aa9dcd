"""The sample that tests/test_gpu_full_graph_train.py checks full-graph training gradients on, without a GPU.

A sparse loss sum(out[S] * w_S) over a seeded destination set S of an L-layer stack depends only on the L-hop
in-neighbourhood R_L of S, so the float64 oracle run on the subgraph induced by R_L (the edges whose destination lies in
R_{L-1}) gives the exact out[S], d node_inp on R_L and every parameter gradient, and the native d node_inp must be
exactly zero outside R_L.  `full_graph_sample` picks S and builds that subgraph; the GPU file imports it.

The point of those tests is the offsets past 2^31: on the ogbn-mag-shaped c2 graph at d = 256 the flat projection
buffer [Q | K'/V'] holds 1.12 x 2^31 fp32 elements, and the bf16 K'/V' table of autocast passes 2^31 bytes.  This file
restates the projection layout on the host and asserts that the sample actually reads rows past both limits, holds hub
destinations on the skewed graph and keeps the 3-hop field small enough for a float64 run, so that a later edit of the
sample cannot quietly drop below 2^31 (the offset twin of the case-list checks in test_gpu_edge_instances.py).
"""
from dataclasses import dataclass

import pytest
import torch

from pyhgt_b200 import synth

TWO31 = 2 ** 31
D = 256                                  # the c2 / c4 width
SAMPLE_COUNTS = (16, 8, 32, 2)           # S per type on the mag-shaped graphs: paper, author, institution, field
SAMPLE_SEED = 5
HUB_PIECE_EDGES = 1024                   # plan.TILE_SPLIT_EDGES (its default; plan.py reads an environment override)


@dataclass
class Sample:
    S: torch.Tensor          # [|S|] sorted node ids whose output rows the loss reads
    reach: list              # reach[k] = R_k, the sorted ids within k in-hops of S (R_0 = S)
    edges: torch.Tensor      # ids of the edges whose destination lies in R_{L-1}: the subgraph's edges
    local: torch.Tensor      # [N] int64: a node's row in the subgraph (its rank in R_L), -1 outside R_L
    sub: synth.HeteroGraph   # the subgraph induced by R_L and `edges`, nodes in id order

    @property
    def nodes(self):
        return self.reach[-1]


def full_graph_sample(g, layers, seed=SAMPLE_SEED, counts=SAMPLE_COUNTS, extra=(), max_in_edges=None):
    """S = `extra` plus counts[t] seeded nodes of each type t (only nodes with at most `max_in_edges` in-edges when that
    is given), then its reach R_1 .. R_L over in-edges and the subgraph the float64 run of an L-layer stack needs."""
    src, dst = g.edge_index[0], g.edge_index[1]
    N = g.num_nodes
    gen = torch.Generator().manual_seed(seed)
    deg = torch.bincount(dst, minlength=N) if max_in_edges is not None else None
    picks = [torch.as_tensor(list(extra), dtype=torch.int64)]
    for t, c in enumerate(counts):
        ids = (g.node_type == t).nonzero(as_tuple=True)[0]
        if deg is not None:
            ids = ids[deg[ids] <= max_in_edges]
        picks.append(ids[torch.randperm(ids.numel(), generator=gen)[:c]])
    S = torch.unique(torch.cat(picks))
    inside = torch.zeros(N, dtype=torch.bool)
    inside[S] = True
    reach, edges = [S], None
    for _ in range(layers):
        edges = inside[dst].nonzero(as_tuple=True)[0]          # the in-edges of R_k
        inside[src[edges]] = True
        reach.append(inside.nonzero(as_tuple=True)[0])
    nodes = reach[-1]
    local = torch.full((N,), -1, dtype=torch.int64)
    local[nodes] = torch.arange(nodes.numel())
    sub = synth.HeteroGraph(g.node_type[nodes], local[g.edge_index[:, edges]], g.edge_type[edges],
                            g.edge_time[edges], g.num_types, g.num_relations, g.name + "-reach%d" % layers)
    return Sample(S, reach, edges, local, sub)


def projection_layout(g, d):
    """Host restatement of the projection buffer of a training layer (plan.build_plan, plan.layer_tables with no active
    prefix and no kv_runs) for a graph whose nodes are sorted by type: the <source type, relation> pairs that occur in
    plan order, the first K'/V' row of each pair, the rows of the K'/V' table without its trailing zero row, and the
    element offset of that table and the buffer's length in the flat [Q | K'/V'] buffer."""
    T, R = g.num_types, g.num_relations
    nt = g.node_type
    assert bool((nt[1:] >= nt[:-1]).all()), "the restatement takes type-sorted node ids (rank == id - type start)"
    counts = torch.bincount(nt, minlength=T).tolist()
    s_t, d_t, r = nt[g.edge_index[0]], nt[g.edge_index[1]], g.edge_type
    ok = (s_t >= 0) & (s_t < T) & (d_t >= 0) & (d_t < T) & (r >= 0) & (r < R)
    present = set(torch.unique(s_t[ok] * R + r[ok]).tolist())
    pairs, pair_row0, rows = [], [], 0
    for s in range(T):
        for rel in range(R):
            if s * R + rel in present:
                pairs.append((s, rel))
                pair_row0.append(rows)
                rows += counts[s]
    kv_off = (g.num_nodes * d + 31) // 32 * 32
    type_row0 = [0]
    for c in counts:
        type_row0.append(type_row0[-1] + c)
    return dict(pairs=pairs, pair_row0=pair_row0, kv_rows=rows, kv_off=kv_off,
                proj_elems=kv_off + (rows + 1) * 2 * d, type_row0=type_row0)


def kv_rows_of(g, layout, edges):
    """The K'/V' table row each of `edges` reads: its <source type, relation> pair's first row plus the source's rank in
    its type (plan.kv_row, in edge-id rather than CSR order)."""
    R = g.num_relations
    src = g.edge_index[0, edges]
    s_t, rel = g.node_type[src], g.edge_type[edges]
    first = torch.full((g.num_types * R,), -1, dtype=torch.int64)
    for (s, r), row0 in zip(layout["pairs"], layout["pair_row0"]):
        first[s * R + r] = row0
    row0 = first[s_t * R + rel]
    assert bool((row0 >= 0).all())
    return row0 + src - torch.as_tensor(layout["type_row0"])[s_t]


def fp32_row_end(layout, rows, d):
    """One past the last element of each fp32 [K'|V'] row in the flat projection buffer."""
    return layout["kv_off"] + (rows + 1) * 2 * d


def bf16_row_end_bytes(rows, d):
    """One past the last byte of each row of the bf16 K'/V' table (autocast), which starts at its own base."""
    return (rows + 1) * 2 * d * 2


def hub_destinations(g, lo=10_000, hi=100_000):
    """(heaviest destination with fewer than `hi` in-edges, another with lo <= in-edges < hi of a different type when one
    exists), and the in-degree of every node."""
    deg = torch.bincount(g.edge_index[1], minlength=g.num_nodes)
    band = ((deg >= lo) & (deg < hi)).nonzero(as_tuple=True)[0]
    first = int(band[deg[band].argmax()])
    others = band[g.node_type[band] != g.node_type[first]]
    others = others if others.numel() else band[band != first]
    second = int(others[deg[others].argmin()])
    return (first, second), deg


@pytest.fixture(scope="module")
def c2():
    return synth.make_mag_shaped(1.0, seed=2)


def test_projection_layout_of_c2_passes_two_to_the_31(c2):
    """The numbers DESIGN.md §5 and the GPU file rely on: the pairs in plan order (paper, cites), (paper, has_topic),
    (author, writes), (author, affiliated_with), and a buffer of 1.12 x 2^31 elements."""
    lay = projection_layout(c2, D)
    assert lay["pairs"] == [(0, 1), (0, 2), (1, 0), (1, 3)]
    assert lay["pair_row0"] == [0, 736_389, 1_472_778, 2_607_427]
    assert lay["kv_rows"] == 3_742_076
    assert lay["kv_off"] == 496_574_208
    assert lay["proj_elems"] == 2_412_517_120 + 2 * D               # + the trailing zero row
    assert lay["proj_elems"] > 1.12 * TWO31
    assert bf16_row_end_bytes(lay["kv_rows"] - 1, D) > 1.78 * TWO31


def test_one_hop_sample_reads_rows_past_two_to_the_31(c2):
    """The sampled edges read fp32 [K'|V'] rows that end past element 2^31 and bf16 rows that end past byte 2^31, and
    rows below both limits too; the subgraph is the destinations' complete in-edge sets."""
    s = full_graph_sample(c2, 1)
    lay = projection_layout(c2, D)
    assert s.S.numel() == sum(SAMPLE_COUNTS)
    rows = kv_rows_of(c2, lay, s.edges)
    past32 = int((fp32_row_end(lay, rows, D) > TWO31).sum())
    past16 = int((bf16_row_end_bytes(rows, D) > TWO31).sum())
    below = int((fp32_row_end(lay, rows, D) <= TWO31).sum())
    assert past32 >= 1000 and past16 >= past32 and below >= 1000, (past32, past16, below)
    assert int(rows.max()) < lay["kv_rows"]
    deg = torch.bincount(c2.edge_index[1], minlength=c2.num_nodes)
    assert s.edges.numel() == int(deg[s.S].sum())
    assert s.sub.num_nodes == s.nodes.numel() and s.sub.num_edges == s.edges.numel()
    assert torch.equal(s.nodes[s.sub.edge_index[1]], c2.edge_index[1, s.edges])
    assert torch.equal(s.nodes[s.sub.edge_index[0]], c2.edge_index[0, s.edges])
    # every type is in S; authors have no in-edges (the update's bias path) and institutions read only author rows
    assert set(c2.node_type[s.S].tolist()) == {0, 1, 2, 3}
    assert int(deg[s.S[c2.node_type[s.S] == 1]].sum()) == 0


def test_three_hop_field_stays_small(c2):
    """The c4 stack's float64 run covers R_3; it must stay a CPU-sized problem and still read past 2^31."""
    s = full_graph_sample(c2, 3)
    assert len(s.reach) == 4 and all(bool(torch.isin(a, b).all()) for a, b in zip(s.reach, s.reach[1:]))
    assert s.nodes.numel() < 100_000, s.nodes.numel()
    assert torch.equal(s.reach[1], full_graph_sample(c2, 1).nodes)
    lay = projection_layout(c2, D)
    assert int((fp32_row_end(lay, kv_rows_of(c2, lay, s.edges), D) > TWO31).sum()) >= 1000


def test_skewed_sample_holds_hub_destinations():
    """On make_mag_shaped(1.0, dst_zipf=1.1) the hub sample holds destinations of 10^4 .. 10^5 in-edges (>= 10 hub
    pieces each) and nothing heavier; the 1.13 M-edge destination stays out (see test_gpu_full_graph_train.py)."""
    g = synth.make_mag_shaped(1.0, seed=2, dst_zipf=1.1)
    (h1, h2), deg = hub_destinations(g)
    assert int(deg.max()) > 1_000_000
    assert 10_000 <= int(deg[h2]) <= int(deg[h1]) < 100_000
    s = full_graph_sample(g, 1, counts=(4, 2, 4, 1), extra=(h1, h2), max_in_edges=HUB_PIECE_EDGES)
    d_s = deg[s.S]
    assert int((d_s >= 10_000).sum()) >= 2 and int(d_s.max()) < 100_000
    assert int(d_s.max()) // HUB_PIECE_EDGES >= 10
    assert int((d_s > HUB_PIECE_EDGES).sum()) == 2                  # the ordinary ones stay below the split threshold
