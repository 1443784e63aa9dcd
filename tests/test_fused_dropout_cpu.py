"""Fused dropout without a GPU: a numpy restatement of the mask contract (include/hgt_b200.h, "Fused dropout"), the
exported symbols, and what ptxas reports for the kernels that draw masks.

`philox4x32_10` is pinned by the known-answer vectors of the Random123 distribution (kat_vectors); `drop_mask` is the
contract on top of it.  tests/test_gpu_fused_dropout.py compares the kernels' masks with it bit for bit, and the kernels
call curand_Philox4x32_10, so that test also ties this file to curand.
"""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np

from pyhgt_b200 import _lib
from pyhgt_b200 import build as hgt_build

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Ten rounds of Philox4x32 over arrays: ctr = (c0, c1, c2, c3), key = (k0, k1), each uint32 [n] -> 4 x uint32 [n]."""
    c = [np.asarray(v, dtype=np.uint64) & U32 for v in ctr]
    k = [np.asarray(v, dtype=np.uint64) & U32 for v in key]
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & U32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & U32]
        k = [(k[0] + np.uint64(W0)) & U32, (k[1] + np.uint64(W1)) & U32]
    return [v.astype(np.uint32) for v in c]


def drop_threshold(p):
    """thr of the contract: the fp32 value of p times 2^32, truncated."""
    return int(float(np.float32(p)) * 4294967296.0)


def drop_scale(p):
    """s = 1 / (1 - p) in fp32; 0 for p >= 1."""
    p32 = np.float32(p)
    return np.float32(0.0) if p32 >= 1 else np.float32(1.0) / (np.float32(1.0) - p32)


def drop_mask(seed, n_rows, d, p):
    """bool [n_rows, d]: element (row, col) is kept iff word col % 4 of Philox(counter = (q, 0, 0), key = seed) >= thr,
    q = row * ceil(d / 4) + col // 4.  p >= 1 keeps nothing."""
    return drop_mask_rows(seed, np.arange(n_rows), d, p)


def drop_mask_rows(seed, rows, d, p):
    """The rows `rows` (rank rows, any order) of drop_mask: bool [len(rows), d].  For masks too large to draw whole,
    such as the sampled rows of a full-graph layer."""
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1)
    if np.float32(p) >= 1:
        return np.zeros((rows.size, d), dtype=bool)
    nchunk = (d + 3) // 4
    q = (rows[:, None] * np.uint64(nchunk) + np.arange(nchunk, dtype=np.uint64)[None, :]).reshape(-1)
    seed = int(seed) & (2 ** 64 - 1)
    zero = np.zeros_like(q)
    words = philox4x32_10((q & U32, q >> np.uint64(32), zero, zero),
                          (np.full_like(q, seed & 0xFFFFFFFF), np.full_like(q, seed >> 32)))
    keep = np.stack(words, 1) >= np.uint32(drop_threshold(p))                   # [rows * nchunk, 4]
    return keep.reshape(rows.size, nchunk * 4)[:, :d]


def test_philox_known_answers():
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = philox4x32_10([[v] for v in ctr], [[v] for v in key])
        assert tuple(int(g[0]) for g in got) == want, (ctr, key, [hex(int(g[0])) for g in got])


def test_mask_contract():
    """The mask is a function of (seed, row, col, d, p): rows do not depend on how many rows are drawn, a column's bit on
    d only through ceil(d / 4); the kept fraction follows 1 - p; seeds and widths give different masks."""
    m = drop_mask(1234567890123, 64, 78, 0.2)
    assert m.shape == (64, 78)
    assert np.array_equal(m[:10], drop_mask(1234567890123, 10, 78, 0.2))
    assert np.array_equal(m[[63, 5, 0, 5]], drop_mask_rows(1234567890123, [63, 5, 0, 5], 78, 0.2))
    assert np.array_equal(m[:, :77], drop_mask(1234567890123, 64, 77, 0.2))     # ceil(78 / 4) == ceil(77 / 4)
    assert not np.array_equal(m[:, :64], drop_mask(1234567890123, 64, 64, 0.2))
    assert not np.array_equal(m, drop_mask(1234567890124, 64, 78, 0.2))
    assert not drop_mask(5, 8, 16, 1.0).any()
    for p in (0.2, 0.5):
        big = drop_mask(99, 4096, 256, p)
        se = (p * (1 - p) / big.size) ** 0.5
        assert abs(big.mean() - (1 - p)) < 5 * se, (p, big.mean())
    # a mask with a larger p is a subset of the mask with a smaller p under the same seed (one threshold on one word)
    assert not (drop_mask(7, 32, 64, 0.5) & ~drop_mask(7, 32, 64, 0.2)).any()
    assert drop_threshold(0.5) == 2 ** 31 and drop_scale(0.5) == 2.0 and drop_scale(1.0) == 0.0


DROP_SYMBOLS = ("hgt_update_epilogue_drop", "hgt_update_backward_drop", "hgt_update_backward_drop_det",
                "hgt_tanh_dropout", "hgt_tanh_dropout_bwd")


def test_fused_dropout_entry_points_are_exported_and_bound():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in DROP_SYMBOLS:
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name
    # the plain twins' arguments, then (seed, p), then the stream
    for plain, drop in (("hgt_update_epilogue", "hgt_update_epilogue_drop"),
                        ("hgt_update_backward", "hgt_update_backward_drop"),
                        ("hgt_update_backward_det", "hgt_update_backward_drop_det")):
        a, b = _lib.SIGNATURES[plain], _lib.SIGNATURES[drop]
        assert b == a[:-1] + [ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p], drop


def test_switch_defaults_off():
    from pyhgt_b200 import DenseHGTConv, HGTConv
    from pyhgt_b200.model import GNN
    assert HGTConv.fused_dropout is False and DenseHGTConv.fused_dropout is False and GNN.fused_dropout is False


def _ptxas_report(src):
    """{mangled kernel name: (spill store bytes, spill load bytes)} of one source of the library, compiled for sm_90a."""
    with tempfile.TemporaryDirectory() as tmp:
        cmd = ([hgt_build._nvcc()] + hgt_build.NVCC_FLAGS +
               ["-Xptxas", "-v", "-c", os.path.join(hgt_build.CSRC, src), "-o", os.path.join(tmp, "out.o")])
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    report = {}
    for m in re.finditer(r"Compiling entry function '(\w+)' for 'sm_90a'.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                         r.stderr, re.S):
        report[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    return report


def test_mask_drawing_kernels_do_not_spill():
    """ptxas -v for sm_90a: the epilogue and tanh kernels that draw masks spill nothing, and neither do the backward
    kernels up to 16 columns per lane (d <= 512).  The 32-column backward instances (d <= 1024) hold five 32-element
    rows per lane at the 255-register limit: their plain twins already spill a few bytes and the mask adds a few more."""
    fwd = _ptxas_report("update.cu")
    drop_fwd = {k: v for k, v in fwd.items() if re.search(r"k_update_epilogue(_vecILi\d+E|I)Lb1E", k) or "k_tanh_dropout" in k}
    assert len(drop_fwd) == 4 + 1 + 4, sorted(drop_fwd)
    assert all(v == (0, 0) for v in drop_fwd.values()), drop_fwd
    bwd = _ptxas_report("update_bwd.cu")
    seen = set()
    for name, spills in bwd.items():
        m = re.search(r"k_update_bwd(_det)?ILi(\d+)ELb1E", name)
        if not m:
            continue
        seen.add((bool(m.group(1)), int(m.group(2))))
        if int(m.group(2)) <= 16:
            assert spills == (0, 0), (name, spills)
        else:
            assert max(spills) <= 64, (name, spills)
    assert seen == {(det, npl) for det in (False, True) for npl in (2, 4, 8, 16, 32)}
