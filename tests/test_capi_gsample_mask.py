"""CPU-side checks of the edge-masked rebuild: the dense rebuild entry points take the mask table where the hashed ones
do and check their arguments, and sample_subgraphs_cuda's edge_mask is validated before anything reaches a device."""
import ctypes

import pytest


def test_rebuild_entry_points_take_the_mask_and_check_their_arguments():
    import __graft_entry__ as ge
    ge.build()
    from pyhgt_b200 import _lib
    lib = _lib.load()
    assert lib.hgt_abi_version() == 5
    for name in ("hgt_gsample_batch_rebuild_count", "hgt_gsample_batch_rebuild_write"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    # dense and hashed rebuild passes take the same arguments, min_ser (NULL: no mask) right after n_blocks
    for name in ("count", "write"):
        dense = _lib.SIGNATURES["hgt_gsample_batch_rebuild_%s" % name]
        assert dense == _lib.SIGNATURES["hgt_gsample_hash_rebuild_%s" % name] and dense[3] is ctypes.c_void_p
    from pyhgt_b200 import sampler
    st = sampler._GBatchState()
    st.num_types, st.n_members = 2, 1
    with pytest.raises(_lib.HgtError, match="batch_rebuild_count"):    # NULL state
        _lib.call("hgt_gsample_batch_rebuild_count", None, None, 0, None, None, 0, 0, None, None, None, None, None, 0,
                  None)
    with pytest.raises(_lib.HgtError, match="batch_rebuild_write"):    # NULL state
        _lib.call("hgt_gsample_batch_rebuild_write", None, None, 0, None, None, None, None, None, None, None, 0, 8, 0,
                  None, 0, None, None, None, None, None, None, None)
    with pytest.raises(_lib.HgtError, match="batch_rebuild_write"):    # NULL member table
        _lib.call("hgt_gsample_batch_rebuild_write", ctypes.byref(st), None, 0, 8, None, None, None, None, None,
                  None, 0, None, 0, None, 0, None, None, None, None, None, None, None)


def test_struct_layouts_are_unchanged():
    from pyhgt_b200 import sampler
    assert ctypes.sizeof(sampler._GBlock) == 5 * 8 + 4 * 4
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
