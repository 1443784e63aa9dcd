"""Layer tables over each type's destination extent (plan.layer_tables(..., dst=True)), host logic only: which rows get Q /
a_linear blocks, which keep only K'/V', and that a plan whose extents cover every row gets the plain tables."""
import numpy as np
import torch

from pyhgt_b200 import plan as P

D = 16


def _plan(counts, pairs, dst_extent):
    T = len(counts)
    type_count = list(counts) + [0]
    type_row0 = [0]
    for c in type_count:
        type_row0.append(type_row0[-1] + c)
    pair_row0, rows = [], 0
    for s, _ in pairs:
        pair_row0.append(rows)
        rows += counts[s]
    N = sum(counts)
    return P.GraphPlan(n_nodes=N, n_edges=0, num_types=T, num_relations=2, has_time=False, sorted_types=True,
                       rank=None, perm=None, type_count=type_count, type_row0=type_row0, type_row0_dev=None,
                       row_ptr=torch.zeros(N + 1, dtype=torch.int32), csr_eid=None, kv_row=None, rte_row=None,
                       pairs=list(pairs), pair_row0=pair_row0, kv_rows=rows, tiles=None, n_tiles=0, n_split=0,
                       dst_extent=list(dst_extent))


def _groups(tab):
    return [tuple(int(v) for v in g) for g in tab[1][:tab[2]]]


def test_extent_tables_cover_q_and_a_linear_rows_up_to_the_extent_only():
    counts, pairs = [3, 4, 6], [(0, 0), (1, 0), (2, 1)]
    p = _plan(counts, pairs, [3, 0, 5])
    lt = P.layer_tables(p, D, D, dst=True)
    assert lt.type_active_dev is None
    assert lt.type_dst_dev.tolist() == [3, 0, 5]
    q_row0 = lt.q_row0
    # (a_row0, m, w_row0, n_cblocks, cb_first, has_bias): type 0 whole, type 1 K'/V' only, type 2 split at its extent
    assert _groups(lt.proj_groups) == [(0, 3, q_row0[0], 3, 0, 1), (3, 4, q_row0[1] + D, 2, 3, 1),
                                       (7, 5, q_row0[2], 3, 5, 1), (12, 1, q_row0[2] + D, 2, 8, 1)]
    assert _groups(lt.upd_groups) == [(0, 3, 0, 1, 0, 1), (7, 5, 2 * D, 1, 1, 1)]
    # bf16 gather tables: a group without a Q block goes to kv_groups whole
    assert [(g[0], g[1]) for g in _groups(lt.q_groups)] == [(0, 3), (7, 5)]
    assert [(g[0], g[1], g[2]) for g in _groups(lt.kv_groups)] == [(0, 3, q_row0[0] + D), (3, 4, q_row0[1] + D),
                                                                  (7, 5, q_row0[2] + D), (12, 1, q_row0[2] + D)]
    # every K'/V' row is still written: the row ranges of each type's K'/V' blocks tile the whole type
    kv_rows = sorted((g[0], g[0] + g[1]) for g in _groups(lt.kv_groups))
    assert kv_rows == [(0, 3), (3, 7), (7, 12), (12, 13)]


def test_full_extents_and_other_modes_keep_the_plain_tables():
    counts, pairs = [3, 4, 6], [(0, 0), (1, 0), (2, 1)]
    full = _plan(counts, pairs, counts)
    assert P.layer_tables(full, D, D, dst=True) is P.layer_tables(full, D, D)
    assert P.layer_tables(full, D, D).type_dst_dev is None
    p = _plan(counts, pairs, [3, 0, 5])
    plain = P.layer_tables(p, D, D)
    assert plain.type_dst_dev is None and plain.type_active_dev is None
    assert _groups(plain.upd_groups) == [(0, 3, 0, 1, 0, 1), (3, 4, D, 1, 1, 1), (7, 6, 2 * D, 1, 2, 1)]
    # sharded runs (active) keep their own tables: the extents do not apply
    act = P.layer_tables(p, D, D, active=[1, 2, 3], dst=True)
    assert act is P.layer_tables(p, D, D, active=[1, 2, 3])
    assert act.type_dst_dev is None and act.type_active_dev.tolist() == [1, 2, 3]
    # sharded-style active tables with the same numbers as the extents are a different entry
    same = P.layer_tables(p, D, D, active=[3, 0, 5])
    assert same is not P.layer_tables(p, D, D, dst=True) and same.type_dst_dev is None


def test_extent_tables_follow_an_overridden_extent():
    counts, pairs = [5, 2], [(0, 0), (1, 1)]
    p = _plan(counts, pairs, [0, 2])
    lt0 = P.layer_tables(p, D, D, dst=True)
    assert lt0.type_dst_dev.tolist() == [0, 2]
    p.dst_extent = [4, 2]
    lt1 = P.layer_tables(p, D, D, dst=True)
    assert lt1 is not lt0 and lt1.type_dst_dev.tolist() == [4, 2]
    p.dst_extent = list(counts)
    assert P.layer_tables(p, D, D, dst=True) is P.layer_tables(p, D, D)
    assert np.array_equal(_groups(P.layer_tables(p, D, D).upd_groups), [(0, 5, 0, 1, 0, 1), (5, 2, D, 1, 1, 1)])
