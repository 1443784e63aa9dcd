"""GPU tests of the persistent typed GEMMs (run on an H100: ``pytest -m gpu``) at group tables large enough that every CTA
of the one-CTA-per-SM grid walks many output tiles, with odd m-tile counts per group and an empty and a one-row group
among them: the forward at BN 256 / 128 / 64 with the fp32 A split by the library and with a presplit A (nothing may be
written outside the column blocks), and the dX / dW backward (also its deterministic entry points, whose dW writes one
partial slot per tile), each against float64."""
import pytest

from pyhgt_b200 import _lib
from tests.test_gpu_bwd import _bwd_case
from tests.test_gpu_parity import _tc_groups_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K,width,spec,act", [
    (256, 256, [(40001, 5), (1, 1), (0, 3), (12345, 3)], None),   # BN 256: 313 and 97 m-tiles, 1857 tiles
    (256, 256, [(40001, 5), (1, 1), (0, 3), (12345, 3)], 1),
    (256, 128, [(20001, 5), (0, 1), (7777, 3)], None),             # BN 128
    (256, 128, [(20001, 5), (0, 1), (7777, 3)], 0),
    (400, 400, [(9999, 3), (1, 1), (5001, 1)], None),              # BN 64, 7 column tiles per block
    (400, 400, [(9999, 3), (1, 1), (5001, 1)], 1),
])
def test_persistent_typed_linear_many_tiles_per_cta_match_fp64(K, width, spec, act):
    err = _tc_groups_case(K, width, spec, act)
    assert err < 5e-5, "max abs err %.3g (relative to max(1, max|ref|))" % err


def test_persistent_typed_linear_bwd_many_tiles_per_cta_match_fp64():
    (ra, ea), (rw, ew), (rb, eb) = _bwd_case(256, 256, [(40001, 5), (1, 1), (0, 3), (12345, 3)], 0, impl=2)
    assert ra < 5e-5, "dA: rel fro %.3g max abs %.3g" % (ra, ea)
    assert rw < 5e-5, "dW: rel fro %.3g max abs %.3g" % (rw, ew)
    assert rb < 1e-5, "db: rel fro %.3g max abs %.3g" % (rb, eb)


def test_persistent_typed_linear_bwd_det_many_tiles_per_cta_repeat_and_match_fp64(monkeypatch):
    """The same case through hgt_typed_linear_bwd_det (same arguments): every per-tile dW slot must be written exactly
    once whichever CTA owns the tile, so two runs agree exactly and both match float64."""
    call = _lib.call

    def det_call(name, *args):
        if name in ("hgt_typed_linear_bwd", "hgt_typed_linear_bwd_workspace_bytes"):
            name = name.replace("hgt_typed_linear_bwd", "hgt_typed_linear_bwd_det")
        return call(name, *args)

    monkeypatch.setattr(_lib, "call", det_call)
    spec = [(40001, 5), (1, 1), (0, 3), (12345, 3)]
    first = _bwd_case(256, 256, spec, 0, impl=2)
    second = _bwd_case(256, 256, spec, 0, impl=2)
    assert first == second, (first, second)
    (ra, ea), (rw, ew), (rb, eb) = first
    assert ra < 5e-5, "dA: rel fro %.3g max abs %.3g" % (ra, ea)
    assert rw < 5e-5, "dW: rel fro %.3g max abs %.3g" % (rw, ew)
    assert rb < 1e-5, "db: rel fro %.3g max abs %.3g" % (rb, eb)
