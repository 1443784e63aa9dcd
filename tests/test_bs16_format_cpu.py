"""The bs16 gather-table format (include/hgt_b200.h, "bs16 gather tables"), restated in numpy.

`encode` / `decode` are the reference the GPU tests compare the producers and the edge kernel against.  Here they are
pinned on the format's guarantees: |m| <= 32767, exact fp32 decoding that never overflows, zero blocks and the zero
row, NaN / Inf blocks, values near FLT_MAX, subnormals, and the 16-byte padding of rows at d = 400.
"""
import numpy as np
import pytest

INV_32767 = np.float32(1.0) / np.float32(32767.0)          # fp32(1 / 32767)
SHRINK = np.float32(1.0 - 2.0 ** -15)                      # r's factor where s >= 2^112
NAN_SCALE = 0x7FC0


def row_bytes(n):
    return (2 * n + n // 8 + 15) // 16 * 16


def scales(x):
    """float32 [rows, n] -> (bf16 scale bits uint32 [rows, n/16], r float32 [rows, n/16]) of every 16-element block."""
    rows, n = x.shape
    amax = (np.ascontiguousarray(x).view(np.uint32).reshape(rows, n // 16, 16) & 0x7FFFFFFF).max(-1)
    t = (amax.view(np.float32) * INV_32767).astype(np.float32)
    sb = ((t.view(np.uint32).astype(np.uint64) + 0xFFFF) >> 16).astype(np.uint32)
    nonfinite = amax >= 0x7F800000
    zero = (sb < 0x80) & ~nonfinite
    sb = np.where(nonfinite, NAN_SCALE, np.where(zero, 0, sb)).astype(np.uint32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        r = (np.float32(1.0) / (sb << 16).view(np.float32)).astype(np.float32)
        r = np.where(sb >= 0x7780, (r * SHRINK).astype(np.float32), r)
    r = np.where(nonfinite | zero, np.float32(0), r).astype(np.float32)
    return sb, r


def mantissas(x):
    """float32 [rows, n] -> (int16 mantissas [rows, n], scale bits [rows, n/16])."""
    rows, n = x.shape
    sb, r = scales(x)
    with np.errstate(invalid="ignore", over="ignore"):
        m = np.rint((x.reshape(rows, n // 16, 16) * r[..., None]).astype(np.float32))
    m = np.where((sb == NAN_SCALE)[..., None], 0, m)
    assert np.abs(m).max(initial=0) <= 32767
    return m.reshape(rows, n).astype(np.int16), sb


def encode(x):
    """float32 [rows, n] (n % 16 == 0) -> uint8 [rows, row_bytes(n)] planar bs16 rows."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, n = x.shape
    m, sb = mantissas(x)
    out = np.zeros((rows, row_bytes(n)), np.uint8)
    out[:, :2 * n] = m.view(np.uint8)
    out[:, 2 * n:2 * n + n // 8] = sb.astype(np.uint16).view(np.uint8)
    return out


def decode(t, n):
    """uint8 [rows, row_bytes(n)] -> float32 [rows, n]: m * s."""
    t = np.ascontiguousarray(t).reshape(-1, row_bytes(n))
    m = t[:, :2 * n].copy().view(np.int16).astype(np.float32)
    s = (t[:, 2 * n:2 * n + n // 8].copy().view(np.uint16).astype(np.uint32) << 16).view(np.float32)
    with np.errstate(invalid="ignore"):
        return (m * np.repeat(s, 16, axis=1)).astype(np.float32)


FLT_MAX = np.finfo(np.float32).max


def test_row_sizes():
    assert [row_bytes(2 * d) for d in (256, 400, 128)] == [1088, 1712, 544]


def test_random_rows_error_and_exact_decode():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((64, 512)) * np.exp(rng.standard_normal((64, 1)) * 20)).astype(np.float32)
    y = decode(encode(x), 512)
    # error at most half a step of the block's scale, which is at most (1 + 2^-7) * max|x| / 32767
    amax = np.abs(x.reshape(64, 32, 16)).max(-1, keepdims=True).astype(np.float64)
    err = np.abs(y.astype(np.float64) - x).reshape(64, 32, 16)
    assert (err <= 0.5 * amax * (1 + 2 ** -7) / 32767 * (1 + 1e-6)).all()
    # m * s is exact: the fp64 product equals the fp32 one
    m, sb = mantissas(x)
    s = np.repeat((sb << 16).view(np.float32), 16, axis=1).astype(np.float64)
    assert np.array_equal(m.astype(np.float64) * s, y.astype(np.float64))


def test_mantissa_bound_is_reached_but_not_passed():
    x = np.zeros((1, 16), np.float32)
    x[0, :] = np.linspace(-1, 1, 16)
    m, sb = mantissas(x)
    assert np.abs(m).max() <= 32767 and np.abs(m).max() > 32767 * (1 - 2 ** -7) - 1


def test_zero_blocks_and_zero_row():
    x = np.zeros((3, 32), np.float32)
    x[1, 16:] = 1.5
    x[2, :] = -0.0
    t = encode(x)
    assert not t[0].any() and not t[2].any()                  # zero (and -0) rows encode to zero bytes
    assert not t[1, :32].any() and not t[1, 64:66].any()      # the zero block of a non-zero row
    assert np.abs(decode(t, 32)[1, 16:] - 1.5).max() < 1.5 / 32767
    assert not np.signbit(decode(t, 32)[2]).any()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_block_decodes_to_nan(bad):
    x = np.ones((1, 48), np.float32)
    x[0, 20] = bad
    t = encode(x)
    y = decode(t, 48)
    assert np.isnan(y[0, 16:32]).all()
    assert np.isfinite(y[0, :16]).all() and np.isfinite(y[0, 32:]).all()
    assert t[0, 96 + 2:96 + 4].view(np.uint16)[0] == NAN_SCALE and not t[0, 32:64].any()


def test_near_flt_max_stays_finite():
    rng = np.random.default_rng(1)
    for k in range(1, 30):
        x = np.full((1, 16), FLT_MAX, np.float32)
        x[0, 1:] = (FLT_MAX * (1 - rng.random(15) * 2.0 ** -k)).astype(np.float32) * np.sign(rng.standard_normal(15))
        y = decode(encode(x), 16)
        assert np.isfinite(y).all(), k
        assert np.abs(y.astype(np.float64) - x).max() <= FLT_MAX * 2.0 ** -14
    x = np.full((1, 16), -FLT_MAX, np.float32)
    assert np.isfinite(decode(encode(x), 16)).all()


def test_subnormals_and_tiny_blocks():
    tiny = np.array([1e-45, 1e-40, 1.17549435e-38, 1e-36, 3.8e-34], np.float32)
    x = np.repeat(tiny[:, None], 16, axis=1)
    x[:, 1::2] *= -1
    sb, _ = scales(x)
    assert (sb[:4] == 0).all()                                # s would be below FLT_MIN: stored as zero
    y = decode(encode(x), 16)
    assert np.isfinite(y).all() and (np.abs(y - x) <= np.abs(x)).all()
    # a subnormal element inside a block of ordinary values rounds to zero or to a multiple of s
    z = np.ones((1, 16), np.float32)
    z[0, 3] = 1e-40
    assert decode(encode(z), 16)[0, 3] == 0


def test_padded_rows_at_d400():
    n = 800
    rng = np.random.default_rng(2)
    x = rng.standard_normal((5, n)).astype(np.float32)
    t = encode(x)
    assert t.shape == (5, 1712) and 2 * n + n // 8 == 1700
    assert not t[:, 1700:].any()
    assert np.abs(decode(t, n) - x).max() < 2 * np.abs(x).max() / 32767
