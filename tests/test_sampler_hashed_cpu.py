"""Host side of the device sampler's hashed state: the layout rule, the region sizes and their growth, and the C-ABI
entry points' argument checks and workspace queries (no device needed)."""
import ctypes as _c

import numpy as np
import pytest

from tests.conftest import load_golden
from tests.test_sampler import _GraphStub


def _sizes(n_ids_row, B, depth, width, n_seed=128, state_room=None):
    from pyhgt_b200 import sampler
    n_ids = np.tile(np.asarray(n_ids_row, dtype=np.int64), (B, 1))
    seeds = np.zeros_like(n_ids)
    seeds[:, 0] = n_seed
    cap = np.minimum(n_ids, seeds + depth * width)
    room = sampler._STATE_ROOM if state_room is None else state_room
    return n_ids, sampler._hash_rooms(n_ids, cap, width, room)


@pytest.mark.parametrize("name", ["sampler", "sampler_large"])
@pytest.mark.parametrize("B", [1, 3, 8, 32])
@pytest.mark.parametrize("depth,width", [(2, 8), (4, 32), (5, 64)])
def test_fixture_sizes_keep_the_dense_state(name, B, depth, width):
    from pyhgt_b200 import sampler
    fg = sampler.FrozenGraph(_GraphStub(load_golden(name)))
    n_ids, rooms = _sizes(list(fg.n_ids.values()), B, depth, width, n_seed=16)
    assert sampler._state_layout(n_ids, rooms, free_bytes=80 << 30) == "dense"


@pytest.mark.parametrize("B", [1, 8, 32])
@pytest.mark.parametrize("depth,width", [(6, 520), (3, 64)])
def test_the_bench_graph_keeps_the_dense_state(B, depth, width):
    """scripts/gpu_sampler_bench.py's MAG-schema graph: 100 k papers, 60 k authors, 8 k fields, 500 venues."""
    from pyhgt_b200 import sampler
    n_ids, rooms = _sizes([100000, 60000, 8000, 500], B, depth, width)
    assert sampler._state_layout(n_ids, rooms, free_bytes=80 << 30) == "dense"


def test_past_the_int32_sort_limit_is_hashed():
    from pyhgt_b200 import sampler
    n_ids, rooms = _sizes([2 ** 31 + 6, 60000, 8000, 500], 8, 4, 32)
    assert sampler._state_layout(n_ids, rooms) == "hashed"
    n_ids, rooms = _sizes([2 ** 28, 60000, 8000, 500], 8, 4, 32)        # 8 x 2^28 ids of one type: 2^31
    assert sampler._state_layout(n_ids, rooms, free_bytes=None) == "hashed"


def test_past_the_memory_share_is_hashed():
    from pyhgt_b200 import sampler
    n_ids, rooms = _sizes([100000, 60000, 8000, 500], 32, 6, 520)
    dense_bytes = sampler._SLOT_BYTES * int(n_ids.sum())
    share = sampler._DENSE_SHARE
    assert sampler._state_layout(n_ids, rooms, free_bytes=int(dense_bytes / share) + 1) == "dense"
    assert sampler._state_layout(n_ids, rooms, free_bytes=int(dense_bytes / share) - 1) == "hashed"


def test_many_more_ids_than_entries_is_hashed():
    from pyhgt_b200 import sampler
    n_ids, rooms = _sizes([100000 * 100, 60000 * 100, 8000 * 100, 500 * 100], 8, 3, 64)
    assert int(n_ids.sum()) > sampler._HASHED_FROM * int(rooms.sum())
    assert sampler._state_layout(n_ids, rooms, free_bytes=80 << 30) == "hashed"


def test_rooms_follow_the_sample_and_stop_at_twice_the_id_range():
    from pyhgt_b200 import sampler
    n_ids = np.array([[10 ** 9, 50, 0]])
    cap = np.array([[128 + 6 * 520, 50, 0]])
    rooms = sampler._hash_rooms(n_ids, cap, 520, 4.0)
    assert rooms.tolist() == [[4 * (128 + 7 * 520), 100, 0]]
    assert sampler._hash_rooms(n_ids, cap, 520, 1e9).tolist() == [[2 * 10 ** 9, 100, 0]]


def test_the_room_grows_on_overflow():
    from pyhgt_b200 import sampler

    class G:
        state_room = sampler._STATE_ROOM

    g = G()
    assert sampler._grow_state_room(g, 0) == 1 and g.state_room == 4 * sampler._STATE_ROOM
    assert sampler._grow_state_room(g, 1) == 2 and g.state_room == 16 * sampler._STATE_ROOM
    n_ids = np.array([[10 ** 6]])
    cap = np.array([[1000]])
    a, b = (sampler._hash_rooms(n_ids, cap, 64, r) for r in (sampler._STATE_ROOM, g.state_room))
    assert b[0, 0] == 16 * a[0, 0]


def test_hash_entry_points_check_their_arguments():
    from pyhgt_b200 import _lib
    _lib.load()
    with pytest.raises(_lib.HgtError, match="hgt_gsample_hash_select_workspace_bytes"):
        _lib.call("hgt_gsample_hash_select_workspace_bytes", 4, 2 ** 31, _c.byref(_c.c_size_t()))
    with pytest.raises(_lib.HgtError, match="hgt_gsample_hash_select_workspace_bytes"):
        _lib.call("hgt_gsample_hash_select_workspace_bytes", 0, 10, _c.byref(_c.c_size_t()))
    for name, n in (("hgt_gsample_hash_insert_seeds", 8), ("hgt_gsample_hash_add_budget", 18),
                    ("hgt_gsample_hash_select", 14), ("hgt_gsample_hash_rebuild_count", 14),
                    ("hgt_gsample_hash_rebuild_write", 22), ("hgt_gsample_hash_rebuild_count_host", 17),
                    ("hgt_gsample_hash_rebuild_write_host", 24)):
        assert len(_lib.SIGNATURES[name]) == n, name
        with pytest.raises(_lib.HgtError, match=name):       # a NULL state
            _lib.call(name, *[None if t is _c.c_void_p else 0 for t in _lib.SIGNATURES[name]])


def test_hash_select_workspace_grows_with_the_entries_not_the_ids():
    from pyhgt_b200 import _lib
    small, big, dense = _c.c_size_t(), _c.c_size_t(), _c.c_size_t()
    _lib.call("hgt_gsample_hash_select_workspace_bytes", 8, 1 << 16, _c.byref(small))
    _lib.call("hgt_gsample_hash_select_workspace_bytes", 8, 1 << 20, _c.byref(big))
    _lib.call("hgt_gsample_batch_select_workspace_bytes", 8, 1 << 20, _c.byref(dense))
    assert 0 < small.value < big.value
    # per entry: the (member, id) keys and entries (2 x 16 B) on top of the dense selection's scratch
    assert big.value >= dense.value + 32 * (1 << 20)
