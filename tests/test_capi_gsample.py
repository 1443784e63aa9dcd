"""CPU-side checks of the device sampler's C entry points (hgt_gsample_*): ABI version, workspace queries, argument
checks, and the ctypes mirrors of its structs."""
import ctypes

import pytest


def test_abi_version_and_workspace_queries():
    import __graft_entry__ as ge
    ge.build()
    from pyhgt_b200 import _lib
    lib = _lib.load()
    assert lib.hgt_abi_version() == 5
    out = ctypes.c_size_t()
    _lib.call("hgt_gsample_batch_add_budget_workspace_bytes", 1, 520, 6, 520, ctypes.byref(out))
    assert out.value >= 3 * 8 * 520 * 6 * 520        # candidate positions, slots and times
    _lib.call("hgt_gsample_batch_select_workspace_bytes", 1, 100000, ctypes.byref(out))
    assert out.value >= 100000 * (2 * 8 + 2 * 4)
    _lib.call("hgt_gsample_rebuild_workspace_bytes", 1000, ctypes.byref(out))
    assert out.value >= 1001 * 8
    with pytest.raises(_lib.HgtError):
        _lib.call("hgt_gsample_batch_add_budget_workspace_bytes", 1, 10, 2, 0, ctypes.byref(out))
    with pytest.raises(_lib.HgtError):
        _lib.call("hgt_gsample_batch_select_workspace_bytes", 1, 2 ** 31, ctypes.byref(out))


def test_struct_mirrors_have_the_c_layout():
    from pyhgt_b200 import sampler
    assert ctypes.sizeof(sampler._GBlock) == 5 * 8 + 4 * 4


def test_device_graph_needs_a_cuda_device():
    from pyhgt_b200 import sampler
    from tests.conftest import load_golden
    from tests.test_sampler import _GraphStub
    with pytest.raises(ValueError):
        sampler.DeviceGraph(sampler.FrozenGraph(_GraphStub(load_golden("sampler"))), "cpu")
