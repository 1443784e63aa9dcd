"""CPU-side checks of the batched device sampler and the disjoint union: the new C entry points, their workspace
queries and argument checks, the ctypes mirrors of the new structs, and merge_batches' host layout logic."""
import ctypes

import numpy as np
import pytest


def test_batched_entry_points_and_workspace_queries():
    import __graft_entry__ as ge
    ge.build()
    from pyhgt_b200 import _lib
    lib = _lib.load()
    assert lib.hgt_abi_version() == 5
    for name in ("hgt_gsample_batch_add_budget", "hgt_gsample_batch_select", "hgt_gsample_batch_rebuild_count",
                 "hgt_gsample_batch_rebuild_write", "hgt_merge_batches"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    many = ctypes.c_size_t()
    # B members need B times the candidate scratch
    _lib.call("hgt_gsample_batch_add_budget_workspace_bytes", 8, 520, 6, 520, ctypes.byref(many))
    assert many.value >= 8 * 3 * 8 * 520 * 6 * 520
    _lib.call("hgt_gsample_batch_select_workspace_bytes", 8, 800000, ctypes.byref(many))
    assert many.value >= 800000 * (2 * 8 + 4 * 4)     # keys, values and the member keys of the second sort pass
    with pytest.raises(_lib.HgtError):
        _lib.call("hgt_gsample_batch_add_budget_workspace_bytes", 0, 10, 2, 8, ctypes.byref(many))
    with pytest.raises(_lib.HgtError):
        _lib.call("hgt_gsample_batch_select_workspace_bytes", 4, 2 ** 31, ctypes.byref(many))
    with pytest.raises(_lib.HgtError):                 # NULL state
        _lib.call("hgt_gsample_batch_select", None, None, None, None, 0, 0, 8, None, None, None, None, None, 0, None)
    with pytest.raises(_lib.HgtError):
        _lib.call("hgt_merge_batches", None, 1, 4, None, None, 0, 0, 0, 0, None, None, None, None, None, None, None)


def test_struct_mirrors_have_the_c_layout():
    from pyhgt_b200 import sampler
    assert ctypes.sizeof(sampler._GBatchState) == 8 + 15 * 8
    assert sampler.MERGE_MEMBER_DTYPE.itemsize == 8 * 8


def test_union_layout_is_type_major():
    from pyhgt_b200 import sampler
    # member 0: 2 papers, 1 author; member 1: 3 papers, 0 authors, 2 venues; member 2: nothing
    tc = [[2, 1, 0], [3, 0, 2], [0, 0, 0]]
    loc_off, uoff, node_base, edge_base, count = sampler.union_layout(tc, [5, 7, 0])
    assert loc_off.tolist() == [[0, 2, 3, 3], [0, 3, 3, 5], [0, 0, 0, 0]]
    assert count.tolist() == [5, 1, 2]
    # type 0 rows: member 0 at 0..1, member 1 at 2..4; type 1: member 0 at 5; type 2: member 1 at 6..7
    assert uoff.tolist() == [[0, 5, 6], [2, 6, 6], [5, 6, 8]]
    assert node_base.tolist() == [0, 3, 8, 8] and edge_base.tolist() == [0, 5, 12, 12]
    # every member row lands on a distinct union row of its own type
    rows, types = [], []
    for b in range(3):
        for t in range(3):
            for i in range(loc_off[b, t], loc_off[b, t + 1]):
                rows.append(uoff[b, t] + i - loc_off[b, t])
                types.append(t)
    assert sorted(rows) == list(range(8))
    assert [types[rows.index(u)] for u in range(8)] == sorted(types)


def test_union_layout_random():
    from pyhgt_b200 import sampler
    rng = np.random.RandomState(0)
    tc = rng.randint(0, 5, (7, 4))
    loc_off, uoff, node_base, _, count = sampler.union_layout(tc, rng.randint(0, 9, 7))
    union_type = np.repeat(np.arange(4), count)
    seen = np.zeros(int(count.sum()), dtype=int)
    for b in range(7):
        for t in range(4):
            u = uoff[b, t] + np.arange(tc[b, t])
            assert (union_type[u] == t).all()
            seen[u] += 1
    assert (seen == 1).all()
    assert node_base[-1] == tc.sum()
