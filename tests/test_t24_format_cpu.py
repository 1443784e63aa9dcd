"""The 24-bit gather-table format (include/hgt_b200.h, "24-bit gather tables") restated in numpy.

`encode` / `decode` are the reference the GPU tests (test_gpu_t24_tables.py) compare the kernels against bitwise; here they
are pinned by hand-picked fp32 bit patterns: ties to even, carries into the exponent, FLT_MAX, +-Inf, NaN, +-0 and
subnormals."""
import numpy as np
import pytest


def round_bits(b):
    """uint32 fp32 words -> rounded words (nearest-even at bit 8, low 8 bits zero; NaN quiet, Inf kept)."""
    b = np.asarray(b, dtype=np.uint32)
    special = (b & np.uint32(0x7F800000)) == np.uint32(0x7F800000)
    nan = special & ((b & np.uint32(0x007FFFFF)) != 0)
    r = ((b.astype(np.uint64) + 0x7F + ((b >> np.uint32(8)) & np.uint32(1))) & 0xFFFFFF00).astype(np.uint32)
    r = np.where(special, b, r)
    return np.where(nan, (b | np.uint32(0x00400000)) & np.uint32(0xFFFFFF00), r).astype(np.uint32)


def encode(x):
    """float32 [..., n] -> uint8 [..., 3n]: planar rows [hi x n (u16, little-endian) | lo x n (u8)]."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    r = round_bits(x.view(np.uint32))
    hi = (r >> np.uint32(16)).astype("<u2").view(np.uint8).reshape(x.shape[:-1] + (2 * x.shape[-1],))
    lo = ((r >> np.uint32(8)) & np.uint32(0xFF)).astype(np.uint8)
    return np.concatenate([hi, lo], axis=-1)


def decode(t):
    """uint8 [..., 3n] -> float32 [..., n]."""
    t = np.ascontiguousarray(t, dtype=np.uint8)
    n = t.shape[-1] // 3
    hi = t[..., :2 * n].copy().view("<u2").astype(np.uint32)
    lo = t[..., 2 * n:].astype(np.uint32)
    return ((hi << np.uint32(16)) | (lo << np.uint32(8))).astype(np.uint32).view(np.float32)


CASES = [
    # (input word, rounded word)
    (0x3F800000, 0x3F800000),   # 1.0: exact
    (0x3F80007F, 0x3F800000),   # below half: down
    (0x3F800080, 0x3F800000),   # tie, kept bit even: down
    (0x3F800180, 0x3F800200),   # tie, kept bit odd: up to even
    (0x3F800081, 0x3F800100),   # above half: up
    (0x3FFFFF80, 0x40000000),   # tie into the exponent: 2.0
    (0x3FFFFFFF, 0x40000000),   # carry into the exponent
    (0xBF800180, 0xBF800200),   # negative tie, odd: magnitude up
    (0x7F7FFFFF, 0x7F800000),   # FLT_MAX rounds past the largest 24-bit value: +Inf
    (0x7F7FFF7F, 0x7F7FFF00),   # just below the halfway point under it: stays finite
    (0xFF7FFFFF, 0xFF800000),   # -FLT_MAX: -Inf
    (0x7F800000, 0x7F800000),   # +Inf
    (0xFF800000, 0xFF800000),   # -Inf
    (0x7F800001, 0x7FC00000),   # signalling NaN with a low payload: still NaN (an add would make it Inf)
    (0xFF800001, 0xFFC00000),   # ... sign kept
    (0x7FC00000, 0x7FC00000),   # quiet NaN
    (0x7FFFFFFF, 0x7FFFFF00),   # NaN with a full payload: low bits dropped, stays NaN
    (0x00000000, 0x00000000),   # +0
    (0x80000000, 0x80000000),   # -0
    (0x00000080, 0x00000000),   # subnormal tie, even: to +0
    (0x00000180, 0x00000200),   # subnormal tie, odd: up
    (0x007FFFFF, 0x00800000),   # largest subnormal carries into the smallest normal
    (0x80000081, 0x80000100),   # negative subnormal
]


@pytest.mark.parametrize("word,want", CASES, ids=["%08x" % w for w, _ in CASES])
def test_round_bits(word, want):
    assert int(round_bits(np.array([word], dtype=np.uint32))[0]) == want


def test_nan_stays_nan_and_inf_stays_inf():
    words = np.array([w for w, _ in CASES], dtype=np.uint32)
    x, r = words.view(np.float32), round_bits(words).view(np.float32)
    assert (np.isnan(x) == np.isnan(r)).all()
    assert (np.isinf(x) <= np.isinf(r)).all()
    assert (np.signbit(x) == np.signbit(r)).all()


def test_planar_layout():
    """Element c of an n-element row: hi at bytes 2c, 2c + 1 (little-endian), lo at byte 2n + c."""
    words = np.array([[0x3F812345, 0xC0ABCDEF, 0x00000000]], dtype=np.uint32)
    t = encode(words.view(np.float32))
    assert t.shape == (1, 9)
    assert list(t[0]) == [0x81, 0x3F, 0xAB, 0xC0, 0x00, 0x00, 0x23, 0xCE, 0x00]
    assert decode(t).view(np.uint32).tolist() == [[0x3F812300, 0xC0ABCE00, 0]]


def test_round_trip_and_error_bound():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((64, 96)) * np.exp(rng.uniform(-20, 20, (64, 96)))).astype(np.float32)
    y = decode(encode(x))
    assert (decode(encode(y)) == y).all()                                   # rounded words encode to themselves
    assert (np.abs(y.astype(np.float64) - x) <= np.abs(x.astype(np.float64)) * 2.0 ** -16).all()
    assert (y.view(np.uint32) == round_bits(x.view(np.uint32))).all()
