"""CPU-side checks of the edge-masked rebuild: the masked entry points exist and check their arguments, the unmasked
ones keep their ABI, and sample_subgraphs_cuda's edge_mask is validated before anything reaches a device."""
import ctypes

import pytest


def test_masked_rebuild_entry_points_and_argument_checks():
    import __graft_entry__ as ge
    ge.build()
    from pyhgt_b200 import _lib
    lib = _lib.load()
    assert lib.hgt_abi_version() == 4
    for name in ("hgt_gsample_batch_rebuild_count_masked", "hgt_gsample_batch_rebuild_write_masked",
                 "hgt_gsample_batch_rebuild_count", "hgt_gsample_batch_rebuild_write"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    # the masked twins take min_ser right after n_blocks; the rest is the unmasked signature
    for name in ("count", "write"):
        plain = _lib.SIGNATURES["hgt_gsample_batch_rebuild_%s" % name]
        twin = _lib.SIGNATURES["hgt_gsample_batch_rebuild_%s_masked" % name]
        assert twin[:3] + twin[4:] == plain and twin[3] is ctypes.c_void_p
    from pyhgt_b200 import sampler
    st = sampler._GBatchState()
    st.num_types, st.n_members = 2, 1
    with pytest.raises(_lib.HgtError, match="count_masked"):           # NULL state
        _lib.call("hgt_gsample_batch_rebuild_count_masked", None, None, 0, None, None, 0, 0, None, None, None, None,
                  None, 0, None)
    with pytest.raises(_lib.HgtError, match="count_masked"):           # NULL mask table
        _lib.call("hgt_gsample_batch_rebuild_count_masked", ctypes.byref(st), None, 0, None, None, 0, 0, None, None,
                  None, None, None, 0, None)
    with pytest.raises(_lib.HgtError, match="write_masked"):           # NULL mask table
        _lib.call("hgt_gsample_batch_rebuild_write_masked", ctypes.byref(st), None, 0, None, None, None, None, None,
                  None, None, 0, 8, 0, None, 0, None, None, None, None, None, None, None)
    with pytest.raises(_lib.HgtError, match="write_masked"):           # NULL member table
        _lib.call("hgt_gsample_batch_rebuild_write_masked", ctypes.byref(st), None, 0, 8, None, None, None, None,
                  None, None, 0, None, 0, None, 0, None, None, None, None, None, None, None)


def test_struct_layouts_are_unchanged():
    from pyhgt_b200 import sampler
    assert ctypes.sizeof(sampler._GBlock) == 5 * 8 + 4 * 4
    assert ctypes.sizeof(sampler._GState) == 8 + 14 * 8
    assert ctypes.sizeof(sampler._GBatchState) == 8 + 15 * 8


class _FakeDeviceGraph:
    """The fields of a DeviceGraph the mask validation reads (no device needed)."""
    types = ["paper", "author", "field"]
    blocks = [(0, 1, "AP_write"), (0, 2, "rev_PF_in_L2"), (0, 0, "self"), (1, 0, "rev_AP_write"),
              (2, 0, "PF_in_L2")]
    n_blocks = 5


def test_edge_mask_table():
    from pyhgt_b200 import sampler
    dg = _FakeDeviceGraph()
    assert sampler._edge_mask_table(dg, None) is None
    assert sampler._edge_mask_table(dg, {}) is None
    tab = sampler._edge_mask_table(dg, {("paper", "field", "rev_PF_in_L2"): (32, 0),
                                        ("field", "paper", "PF_in_L2"): (0, 32)})
    assert tab.tolist() == [0, 0, 32, 0, 0, 0, 0, 0, 0, 32]
    with pytest.raises(KeyError):                                       # not a block of the graph
        sampler._edge_mask_table(dg, {("paper", "venue", "rev_PV_Journal"): (4, 0)})
    with pytest.raises(KeyError):
        sampler._edge_mask_table(dg, {("paper", "field"): (4, 0)})
    with pytest.raises(ValueError):                                     # self loops are never masked
        sampler._edge_mask_table(dg, {("paper", "paper", "self"): (4, 0)})
    with pytest.raises(ValueError):
        sampler._edge_mask_table(dg, {("paper", "author", "AP_write"): (-1, 0)})
    with pytest.raises(ValueError):
        sampler._edge_mask_table(dg, {("paper", "author", "AP_write"): (0, -3)})
