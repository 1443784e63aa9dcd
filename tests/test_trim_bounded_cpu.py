"""CPU-side checks of the bounded hop layout: TrimSignature arithmetic (bounds -> active prefixes, K'/V' runs, adapter
rows, row count) and hgt_trim_layout_bounded's argument checks, which fire before anything reaches a device."""
import numpy as np
import pytest


def _lib():
    import __graft_entry__ as ge
    ge.build()
    from pyhgt_b200 import _lib
    _lib.load()
    return _lib


def test_signature_validates_and_sizes_rows():
    from pyhgt_b200 import trim
    b = [[3, 5, 0, 7], [1, 0, 2, 0]]
    s = trim.TrimSignature(b, 2)
    assert s.num_types == 2 and s.n_layers == 2
    assert s.n_rows == 18 + 1                                     # every slot plus the pad row
    assert s.key() == trim.TrimSignature(np.asarray(b, dtype=np.int32), 2).key()
    assert s.key() != trim.TrimSignature([[3, 5, 1, 7], [1, 0, 2, 0]], 2).key()
    with pytest.raises(ValueError):
        trim.TrimSignature(b, 3)                                  # L+2 columns
    with pytest.raises(ValueError):
        trim.TrimSignature([[1, -1, 0, 0]], 2)
    with pytest.raises(ValueError):
        trim.TrimSignature([[1, 2]], 0)
    with pytest.raises(ValueError):
        trim.TrimSignature([[2 ** 31, 0, 0]], 1)


def test_views_from_hand_made_bounds():
    """The host arithmetic of build_layout on bounds: layer l computes the rows of hop classes 0..L-l of every type,
    reads K'/V' over 0..L-l+1, the adapter covers 0..L; each type's rows are the sum of its bounds."""
    from pyhgt_b200 import trim
    bounds = [[2, 3, 4, 5, 6], [1, 0, 0, 2, 9], [0, 1, 1, 1, 0]]               # L = 3
    type_rows, actives, kvs, adapter = trim.slot_prefixes(bounds)
    assert type_rows == [20, 12, 3]
    assert actives == [(9, 1, 2), (5, 1, 1), (2, 1, 0)]                          # layers 1, 2, 3
    assert kvs == [(14, 3, 3), (9, 1, 2), (5, 1, 1)]
    assert adapter == (14, 3, 3)
    type_rows, actives, kvs, adapter = trim.slot_prefixes([[4, 1, 7]])          # L = 1
    assert (type_rows, actives, kvs, adapter) == ([12], [(4,)], [(5,)], (5,))


def test_bounded_entry_point_argument_checks():
    lib = _lib()
    assert lib.load().hgt_abi_version() == 5
    assert "hgt_trim_layout_bounded" in lib.SIGNATURES and hasattr(lib.load(), "hgt_trim_layout_bounded")
    assert len(lib.SIGNATURES["hgt_trim_layout_bounded"]) == len(lib.SIGNATURES["hgt_trim_layout"]) + 2
    T, R, L, N, E = 2, 3, 2, 10, 0
    fake = 4096                                                   # never dereferenced: every call fails its checks first
    good = np.array([[1, 2, 0, 0], [3, 0, 1, 0]], dtype=np.int32)

    def call(bounds, n_rows, T=T, L=L, meta=fake):
        ptr = None if bounds is None else bounds.ctypes.data
        lib.call("hgt_trim_layout_bounded", None, None, None, fake, N, E, T, R, None, 0, L, ptr, n_rows,
                 fake, fake, fake, fake, None, None, meta, None, 1 << 40, None)

    with pytest.raises(lib.HgtError, match="NULL hop_bounds"):
        call(None, 8)
    with pytest.raises(lib.HgtError, match="unsupported"):
        call(good, 8, L=0)
    with pytest.raises(lib.HgtError, match="unsupported"):
        call(good, 8, T=0)
    with pytest.raises(lib.HgtError, match="NULL argument"):
        call(good, 8, meta=None)
    neg = good.copy()
    neg[1, 2] = -1
    with pytest.raises(lib.HgtError, match="negative"):
        call(neg, 8)
    with pytest.raises(lib.HgtError, match="below the sum"):
        call(good, 6)                                             # the bounds sum to 7
    with pytest.raises(lib.HgtError, match="at least 1"):
        call(np.zeros((T, L + 2), dtype=np.int32), 0)
    with pytest.raises(lib.HgtError, match="out of range"):
        call(good, -1)
