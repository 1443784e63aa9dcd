"""torch.set_float32_matmul_precision("medium") -> one bf16 product in the typed GEMMs: the parts that need no device.

The precision reader maps every torch setting, gemm_impl keeps SIMT where the layer asked for it, and the workspace
queries (host arithmetic only) accept impl 3, answer no more than impl 2 and reject an unknown impl.
"""
import ctypes

import numpy as np
import pytest
import torch

from pyhgt_b200 import _lib
from pyhgt_b200.autograd import bf16_matmuls, gemm_impl


@pytest.fixture
def restore_precision():
    old = torch.get_float32_matmul_precision()
    yield
    torch.set_float32_matmul_precision(old)


@pytest.mark.parametrize("setting, one", [("highest", False), ("high", False), ("medium", True)])
def test_reader_maps_each_setting(restore_precision, setting, one):
    torch.set_float32_matmul_precision(setting)
    assert bf16_matmuls() is one


def test_gemm_impl():
    assert [gemm_impl(i, False) for i in (0, 1, 2)] == [0, 1, 2]
    assert [gemm_impl(i, True) for i in (0, 1, 2)] == [3, 1, 3]


def _groups(ms, ncb, width):
    g = np.zeros(len(ms), dtype=_lib.LIN_GROUP_DTYPE)
    c = np.zeros(len(ms) * ncb, dtype=_lib.LIN_CBLOCK_DTYPE)
    a0 = out0 = 0
    for i, m in enumerate(ms):
        g[i] = (a0, m, i * ncb * width, ncb, i * ncb, 1)
        for cb in range(ncb):
            c[i * ncb + cb] = (out0 + cb * width, ncb * width)
        a0 += m
        out0 += m * ncb * width
    return g, c, out0


SHAPES = [(256, 256, (736, 1134, 87), 5), (400, 400, (3000, 17), 1), (128, 256, (5000,), 2), (64, 24, (900,), 1)]


def _fwd_bytes(g, K, width, impl):
    b = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g.ctypes.data, len(g), K, width, impl, ctypes.byref(b))
    return b.value


def _bwd_bytes(g, c, K, width, elems, impl, dsplit=0, asplit=0):
    b = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_bwd_workspace_bytes", g.ctypes.data, len(g), c.ctypes.data, K, width, K, elems, dsplit,
              asplit, impl, ctypes.byref(b))
    return b.value


@pytest.mark.parametrize("K, width, ms, ncb", SHAPES)
def test_forward_workspace_query(K, width, ms, ncb):
    g, _, _ = _groups(ms, ncb, width)
    one, three = _fwd_bytes(g, K, width, 3), _fwd_bytes(g, K, width, 2 if width % 16 == 0 else 1)
    assert one <= three
    if width % 16 == 0:
        assert one < three                                # no lo halves of A and W
    else:
        assert one == 0 == _fwd_bytes(g, K, width, 0)     # auto picks SIMT, and so does impl 3
    with pytest.raises(_lib.HgtError, match="unknown impl 4"):
        _fwd_bytes(g, K, width, 4)


@pytest.mark.parametrize("K, width, ms, ncb", SHAPES)
def test_backward_workspace_query(K, width, ms, ncb):
    g, c, elems = _groups(ms, ncb, width)
    for dsplit, asplit in ((0, 0), (1, 0), (0, 1), (1, 1)):
        assert _bwd_bytes(g, c, K, width, elems, 3, dsplit, asplit) <= _bwd_bytes(g, c, K, width, elems, 2, dsplit, asplit)
    with pytest.raises(_lib.HgtError, match="unknown impl 4"):
        _bwd_bytes(g, c, K, width, elems, 4)
