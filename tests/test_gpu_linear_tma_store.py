"""The forward typed GEMM's asynchronous TMA tensor-store epilogue (tcp::store_tma) against its staged st.global epilogue
(tcp::store_staged), bitwise.

At 128- and 256-column tiles the kernel takes the tensor-store path when a tile's destination rows are 16-byte aligned,
and falls back to the staged path when they are not.  Each case runs the same product twice: into an aligned output, and
into the same buffer shifted by one element (every row misaligned, so every tile takes the fallback).  Both must write the same bits, including the clipped
group tails and the columns past a column block, and leave the elements around the output untouched.
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
    """Groups of m rows with `ncb` column blocks each; a group's blocks sit side by side in rows of ld = ncb * width +
    pad elements."""
    groups, cblocks, a0, out0, w0 = [], [], 0, 0, 0
    ld = ncb * width + pad
    for g, m in enumerate(ms):
        groups.append((a0, m, w0, ncb, len(cblocks), g % 3 != 1))
        cblocks += [(out0 + cb * width, ld) for cb in range(ncb)]
        a0 += m
        out0 += m * ld
        w0 += ncb * width
    return P._pack_groups(groups, cblocks, _dev()), a0, out0, w0


class _Case:
    def __init__(self, K, width, ms, ncb, pad, presplit, seed=0):
        dev = _dev()
        self.K, self.width, self.presplit = K, width, presplit
        self.tab, self.rows, self.out_elems, w_rows = _table(width, ms, ncb, pad)
        gen = torch.Generator().manual_seed(seed + K + width + len(ms) + ncb + pad)
        self.a = (torch.randn(self.rows, K, generator=gen) * 2).to(dev)
        self.w = torch.randn(w_rows, K, generator=gen).to(dev)
        self.b = torch.randn(w_rows, generator=gen).to(dev)
        g_host, n_g = self.tab[1], self.tab[2]
        wsb = ctypes.c_size_t()
        if presplit:
            self.hi = torch.empty(self.rows, K, dtype=BF16, device=dev)
            self.lo = torch.empty(self.rows, K, dtype=BF16, device=dev)
            _lib.call("hgt_act_split", self.a.data_ptr(), K, self.rows, K, 0, None, self.hi.data_ptr(),
                      self.lo.data_ptr(), _st())
            _lib.call("hgt_typed_linear_presplit_workspace_bytes", g_host.ctypes.data, n_g, K, width, ctypes.byref(wsb))
        else:
            _lib.call("hgt_typed_linear_workspace_bytes", g_host.ctypes.data, n_g, K, width, 2, ctypes.byref(wsb))
        self.ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=dev)

    def run(self, out):
        g_dev, g_host, n_g, c_dev = self.tab
        bf16 = out.dtype == BF16
        if self.presplit:
            fn = "hgt_typed_linear_presplit_bf16" if bf16 else "hgt_typed_linear_presplit"
            _lib.call(fn, self.hi.data_ptr(), self.lo.data_ptr(), self.w.data_ptr(), self.b.data_ptr(), self.K,
                      self.width, g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), out.data_ptr(),
                      self.ws.data_ptr(), self.ws.numel(), _st())
        else:
            fn = "hgt_typed_linear_bf16" if bf16 else "hgt_typed_linear"
            _lib.call(fn, self.a.data_ptr(), self.K, self.w.data_ptr(), self.b.data_ptr(), self.K, self.width,
                      g_dev.data_ptr(), g_host.ctypes.data, n_g, c_dev.data_ptr(), out.data_ptr(), 2,
                      self.ws.data_ptr(), self.ws.numel(), _st())

    def aligned_and_shifted(self, dtype):
        """(output written at a 16-byte aligned address, the same output written one element further on)."""
        buf = torch.full((self.out_elems + 16,), SENTINEL, dtype=dtype, device=_dev())
        shifted = torch.full((self.out_elems + 16,), SENTINEL, dtype=dtype, device=_dev())
        assert buf.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 0
        self.run(buf[8:])
        self.run(shifted[9:])
        torch.cuda.synchronize()
        return buf, shifted


def _bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def _check(case, dtype):
    buf, shifted = case.aligned_and_shifted(dtype)
    got, ref = buf[8:8 + case.out_elems], shifted[9:9 + case.out_elems]
    assert torch.equal(_bits(got), _bits(ref))
    # nothing written outside the output
    assert bool((buf[:8] == SENTINEL).all()) and bool((buf[8 + case.out_elems:] == SENTINEL).all())
    assert bool((shifted[:9] == SENTINEL).all()) and bool((shifted[9 + case.out_elems:] == SENTINEL).all())
    return got


def _fp64_ref(case, ms, ncb, pad):
    """The fp32 output recomputed in float64 from the same operands (padding columns left at the sentinel)."""
    ld = ncb * case.width + pad
    out = torch.full((case.out_elems,), SENTINEL, dtype=torch.float64, device=_dev())
    a0 = out0 = w0 = 0
    a, w, b = case.a.double(), case.w.double(), case.b.double()
    for g, m in enumerate(ms):
        blk = a[a0:a0 + m] @ w[w0:w0 + ncb * case.width].T
        if g % 3 != 1:
            blk = blk + b[w0:w0 + ncb * case.width]
        view = out[out0:out0 + m * ld].view(m, ld)
        view[:, :ncb * case.width] = blk
        a0, out0, w0 = a0 + m, out0 + m * ld, w0 + ncb * case.width
    return out


TAILS = [1, 63, 64, 65, 127]


@pytest.mark.parametrize("presplit", [False, True], ids=["split", "presplit"])
@pytest.mark.parametrize("dtype", [torch.float32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("K,width,ncb,pad", [
    (64, 64, 2, 0),       # BN = 64 (staged epilogue either way)
    (96, 128, 3, 0),      # BN = 128
    (128, 256, 2, 0),     # BN = 256
    (64, 80, 3, 0),       # BN = 128, the last 48 columns of each tile past the column block
    (64, 400, 2, 0),      # BN = 64
    (128, 256, 2, 16),    # padded ld
    (64, 80, 2, 8),       # padded ld, clipped columns
])
def test_tma_store_equals_staged_store(K, width, ncb, pad, dtype, presplit):
    ms = [128 * (i % 3) + t for i, t in enumerate(TAILS)]
    case = _Case(K, width, ms, ncb, pad, presplit)
    got = _check(case, dtype)
    if dtype == torch.float32:
        ref = _fp64_ref(case, ms, ncb, pad)
        scale = float(ref.abs().max())
        assert float((got.double() - ref).abs().max()) <= 5e-5 * scale


@pytest.mark.parametrize("presplit", [False, True], ids=["split", "presplit"])
@pytest.mark.parametrize("dtype", [torch.float32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("width", [128, 256])
def test_tma_store_equals_staged_store_many_groups(width, dtype, presplit):
    """More than 64 groups: the launches are chunked, and each chunk rebuilds the output maps the previous chunk used."""
    ms = [1 + 37 * i for i in range(70)]
    case = _Case(64, width, ms, 2, 0, presplit)
    _check(case, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, BF16], ids=["fp32", "bf16"])
def test_tma_store_projection_replays_from_a_cuda_graph(dtype):
    """A c2-shaped projection (K = 256, 256-wide column blocks, Q + K' + V' per type) captured in a CUDA graph: the replay,
    with new operand values, equals an eager call on the same values."""
    ms = [20000 + 65, 9000 + 1, 3000 + 127]
    case = _Case(256, 256, ms, 3, 0, presplit=True, seed=5)
    out = torch.full((case.out_elems,), SENTINEL, dtype=dtype, device=_dev())
    case.run(out)                                             # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        case.run(out)
    gen = torch.Generator().manual_seed(11)
    case.w.copy_(torch.randn(case.w.shape, generator=gen))
    a = torch.randn(case.a.shape, generator=gen).to(_dev())
    _lib.call("hgt_act_split", a.data_ptr(), case.K, case.rows, case.K, 0, None, case.hi.data_ptr(),
              case.lo.data_ptr(), _st())
    out.fill_(SENTINEL)
    g.replay()
    torch.cuda.synchronize()
    eager = torch.full_like(out, SENTINEL)
    case.run(eager)
    torch.cuda.synchronize()
    assert bool((out != SENTINEL).any())
    assert torch.equal(_bits(out), _bits(eager))
