"""C-ABI symbols of the deterministic training backward (CPU: needs the built library, not a GPU)."""
import ctypes

from pyhgt_b200 import _lib

DET_SYMBOLS = ("hgt_plan_source_index", "hgt_edge_backward_det_workspace_bytes", "hgt_edge_backward_dst",
               "hgt_edge_backward_rows", "hgt_typed_linear_bwd_det_workspace_bytes", "hgt_typed_linear_bwd_det",
               "hgt_update_backward_det_workspace_bytes", "hgt_update_backward_det", "hgt_fold_backward_det")


def test_deterministic_entry_points_are_exported_and_bound():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in DET_SYMBOLS:
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name
    lib.hgt_abi_version.restype = ctypes.c_int
    assert lib.hgt_abi_version() >= 3


def test_deterministic_workspace_sizes_on_the_host():
    """The workspace queries are host-only: they work without a device and grow with the partial slots they count."""
    _lib.load()
    b = ctypes.c_size_t()
    _lib.call("hgt_edge_backward_det_workspace_bytes", 10, 3, 64, ctypes.byref(b))
    assert b.value == 256 + 4 * max(10 * 64, 3 * 2 * 64)
    _lib.call("hgt_update_backward_det_workspace_bytes", 1000, 3, 64, ctypes.byref(b))
    assert b.value == ((1000 + 511) // 512 + 3 + 1) * (2 * 64 + 1) * 4
