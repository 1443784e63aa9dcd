"""The forward typed GEMM's workspace holds W's bf16 halves and the output maps, not halves of A.

At 128- and 256-column tiles the tensor-core GEMM splits fp32 A as it loads it, so hgt_typed_linear_workspace_bytes (and
the presplit query) must not grow with the groups' row counts.  64-column tiles still read A split up front and keep its
halves there; the SIMT path needs no workspace at all.  Host arithmetic only.
"""
import ctypes

import numpy as np
import pytest

from pyhgt_b200 import _lib


def _groups(ms, ncb, width):
    g = np.zeros(len(ms), dtype=_lib.LIN_GROUP_DTYPE)
    a0 = 0
    for i, m in enumerate(ms):
        g[i] = (a0, m, i * ncb * width, ncb, i * ncb, 1)
        a0 += m
    return g


def _bytes(fn, g, K, width, *impl):
    b = ctypes.c_size_t()
    _lib.call(fn, g.ctypes.data, len(g), K, width, *impl, ctypes.byref(b))
    return b.value


C2_ROWS = (736389, 1134649, 8740, 59965)


@pytest.mark.parametrize("K, width, ncb", [(256, 256, 5), (400, 256, 2), (128, 128, 3), (64, 80, 1)])
@pytest.mark.parametrize("impl", [2, 3])
def test_forward_workspace_independent_of_rows(K, width, ncb, impl):
    small = _groups([r // 1000 + 1 for r in C2_ROWS], ncb, width)
    big = _groups([r * 3 for r in C2_ROWS], ncb, width)
    a = _bytes("hgt_typed_linear_workspace_bytes", small, K, width, impl)
    b = _bytes("hgt_typed_linear_workspace_bytes", big, K, width, impl)
    assert a == b
    halves = 1 if impl == 3 else 2
    w_rows = len(C2_ROWS) * ncb * width
    assert b < halves * w_rows * K * 2 + 128 * len(C2_ROWS) * ncb + 4096      # W's halves + output maps + alignment
    assert _bytes("hgt_typed_linear_presplit_workspace_bytes", small, K, width) == \
        _bytes("hgt_typed_linear_presplit_workspace_bytes", big, K, width)


@pytest.mark.parametrize("impl", [2, 3])
def test_64_column_tiles_keep_a_halves(impl):
    K = width = 400                                           # d = 400: 64-column tiles
    small, big = _groups([1000], 2, width), _groups([101000], 2, width)
    grow = _bytes("hgt_typed_linear_workspace_bytes", big, K, width, impl) - \
        _bytes("hgt_typed_linear_workspace_bytes", small, K, width, impl)
    assert grow == (1 if impl == 3 else 2) * 100000 * K * 2


def test_simt_needs_no_workspace():
    g = _groups(C2_ROWS, 1, 24)
    assert _bytes("hgt_typed_linear_workspace_bytes", g, 64, 24, 1) == 0
    assert _bytes("hgt_typed_linear_workspace_bytes", g, 64, 24, 0) == 0       # width % 16 != 0: auto takes SIMT
