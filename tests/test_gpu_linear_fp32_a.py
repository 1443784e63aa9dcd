"""The forward typed GEMM reading fp32 A and splitting it in shared memory, against the same GEMM fed A already split.

At 128- and 256-column tiles hgt_typed_linear[_bf16] loads fp32 A with TMA and each consumer warpgroup splits its rows
into bf16 hi + lo itself (64-column tiles read A split by a k_split_bf16 pass first);
hgt_typed_linear_presplit[_bf16] reads hi / lo that hgt_act_split wrote.  The halves are the same round-to-nearest bits
and the products run in the same order, so the two must agree bitwise: every tile width (BN = 64 / 128 / 256), fp32 and
bf16 output, three products and one (impl 3, torch's "medium" matmul precision), K that is and is not a multiple of the
32- or 64-wide k-block, group tails, column blocks past the tile, a strided A, and the c2 projection's group table at
reduced row counts.  An A that TMA cannot load as fp32 (base not 16-byte aligned, or lda % 4 != 0) is split by a separate
pass first and must give the same bits too.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from pyhgt_b200 import _lib, plan as P          # noqa: E402

BF16 = torch.bfloat16
SENTINEL = -7.0


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _table(width, ms, ncb, pad):
    """Groups of m rows with `ncb` column blocks each, side by side in output rows of ld = ncb * width + pad."""
    groups, cblocks, a0, out0, w0 = [], [], 0, 0, 0
    ld = ncb * width + pad
    for g, m in enumerate(ms):
        groups.append((a0, m, w0, ncb, len(cblocks), g % 3 != 1))
        cblocks += [(out0 + cb * width, ld) for cb in range(ncb)]
        a0 += m
        out0 += m * ld
        w0 += ncb * width
    return P._pack_groups(groups, cblocks, _dev()), a0, out0, w0


def _bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def _run(K, width, ms, ncb, pad=0, dtype=torch.float32, one=False, lda=None, offset=0, seed=0):
    """(fp32-A output, presplit output, kernels the fp32-A call launched, kernels the presplit call launched)."""
    dev = _dev()
    lda = K if lda is None else lda
    tab, rows, out_elems, w_rows = _table(width, ms, ncb, pad)
    g_dev, g_host, n_g, c_dev = tab
    gen = torch.Generator().manual_seed(seed + 7 * K + width + len(ms) + ncb + pad + lda + offset)
    # A lives `offset` floats into its buffer, rows lda apart; the columns past K hold values that must not be read
    buf = (torch.randn(offset + rows * lda + 4, generator=gen) * 3).to(dev)
    a = buf[offset:offset + rows * lda].view(rows, lda)
    w = torch.randn(w_rows, K, generator=gen).to(dev)
    b = torch.randn(w_rows, generator=gen).to(dev)
    hi = torch.empty(rows, K, dtype=BF16, device=dev)
    lo = None if one else torch.empty(rows, K, dtype=BF16, device=dev)
    _lib.call("hgt_act_split", a.data_ptr(), lda, rows, K, 0, None, hi.data_ptr(), _lib.ptr(lo), _st())

    wsb = ctypes.c_size_t()
    _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, 3 if one else 2, ctypes.byref(wsb))
    ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)
    _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
    ws_pre = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)

    got = torch.full((out_elems,), SENTINEL, dtype=dtype, device=dev)
    ref = torch.full((out_elems,), SENTINEL, dtype=dtype, device=dev)
    sfx = "_bf16" if dtype == BF16 else ""
    torch.cuda.synchronize()
    n0 = _lib.kernel_launches()
    _lib.call("hgt_typed_linear" + sfx, a.data_ptr(), lda, w.data_ptr(), b.data_ptr(), K, width, g_dev.data_ptr(),
              g_host.ctypes.data, n_g, c_dev.data_ptr(), got.data_ptr(), 3 if one else 2, ws.data_ptr(), ws.numel(),
              _st())
    n1 = _lib.kernel_launches()
    _lib.call("hgt_typed_linear_presplit" + sfx, hi.data_ptr(), _lib.ptr(lo), w.data_ptr(), b.data_ptr(), K, width,
              g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), ref.data_ptr(), ws_pre.data_ptr(),
              ws_pre.numel(), _st())
    n2 = _lib.kernel_launches()
    torch.cuda.synchronize()
    return got, ref, n1 - n0, n2 - n1


def _check(*args, **kw):
    got, ref, n_f32, n_pre = _run(*args, **kw)
    assert bool((ref != SENTINEL).any())
    assert torch.equal(_bits(got), _bits(ref))
    return n_f32, n_pre


def _split_passes(width):
    """Passes over A before the fp32-A call's GEMM: one at 64-column tiles, none at 128 / 256 (the tile width pads
    `width` least, ties to the wider tile, as tcp::pick_tile_n)."""
    pads = {bn: -(-width // bn) * bn for bn in (64, 128, 256)}
    return 1 if pads[64] < min(pads[128], pads[256]) else 0


TAILS = [1, 63, 64, 65, 127]
DTYPES = pytest.mark.parametrize("dtype", [torch.float32, BF16], ids=["fp32", "bf16"])
PRODUCTS = pytest.mark.parametrize("one", [False, True], ids=["x3", "x1"])


@PRODUCTS
@DTYPES
@pytest.mark.parametrize("K,width,ncb,pad", [
    (64, 64, 2, 0),       # BN = 64
    (128, 400, 1, 0),     # BN = 64, the last 16 columns past the column block
    (400, 400, 2, 0),     # BN = 64, K = 400: a k-block past K (zero-filled by TMA)
    (64, 128, 3, 0),      # BN = 128
    (256, 80, 3, 0),      # BN = 128, the last 48 columns of each tile past the column block
    (400, 128, 1, 0),     # BN = 128, K = 400 not a multiple of the 32-wide k-block
    (128, 256, 2, 0),     # BN = 256
    (256, 256, 2, 16),    # BN = 256, padded ld
    (400, 256, 1, 0),     # BN = 256, K = 400
    (64, 80, 2, 8),       # padded ld, clipped columns
])
def test_fp32_a_equals_presplit(K, width, ncb, pad, dtype, one):
    ms = [128 * (i % 3) + t for i, t in enumerate(TAILS)]
    n_f32, n_pre = _check(K, width, ms, ncb, pad, dtype=dtype, one=one)
    assert n_f32 == n_pre + _split_passes(width)


@PRODUCTS
@DTYPES
@pytest.mark.parametrize("K,width", [(64, 64), (128, 256), (400, 128)])
def test_fp32_a_strided(K, width, dtype, one):
    """lda > K: the columns between K and lda are neither read nor allowed to reach the products."""
    n_f32, n_pre = _check(K, width, [300, 77], 2, dtype=dtype, one=one, lda=K + 12)
    assert n_f32 == n_pre + _split_passes(width)


@PRODUCTS
@DTYPES
def test_fp32_a_c2_projection_table(dtype, one):
    """The c2 projection's groups (736,389 / 1,134,649 / 8,740 / 59,965 rows, five 256-wide column blocks, K = 256) at
    about 1 / 100 of the rows, group tails kept."""
    _check(256, 256, [7364, 11347, 87, 600], 5, dtype=dtype, one=one)


@PRODUCTS
@DTYPES
@pytest.mark.parametrize("lda,offset", [(128, 1), (129, 0)], ids=["base+4B", "lda%4"])
def test_fp32_a_unloadable_takes_the_split_pass(lda, offset, dtype, one):
    n_f32, n_pre = _check(128, 256, [300, 77], 2, dtype=dtype, one=one, lda=lda, offset=offset)
    assert n_f32 == n_pre + 1                                 # k_split_bf16 over A first


def test_fp32_a_many_groups():
    """More than 64 groups: chunked launches, each splitting its own rows."""
    n_f32, n_pre = _check(64, 256, [1 + 37 * i for i in range(70)], 2)
    assert n_f32 == n_pre
