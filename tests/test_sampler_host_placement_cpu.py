"""DeviceGraph(..., placement="host") without a GPU: the placement check comes before any CUDA call, the hit-record
scratch of the single-read rebuild is sized and grown on the host, and the new C entry points reject bad arguments
before they touch CUDA."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_sampler import _GraphStub
from tests.conftest import load_golden


@pytest.mark.parametrize("bad", ["pinned", "Host", "", None, 1])
def test_bad_placement_raises_value_error_before_cuda(bad):
    from pyhgt_b200 import sampler
    fg = sampler.FrozenGraph(_GraphStub(load_golden("sampler")))
    was = torch.cuda.is_initialized()
    with pytest.raises(ValueError, match="placement"):
        sampler.DeviceGraph(fg, "cuda:0", placement=bad)
    assert torch.cuda.is_initialized() == was


def test_placements_and_default():
    import inspect
    from pyhgt_b200 import sampler
    assert sampler.DeviceGraph.PLACEMENTS == ("device", "host")
    assert inspect.signature(sampler.DeviceGraph).parameters["placement"].default == "device"


class _Room:
    hit_room = 8.0


def test_hit_capacity_scales_with_the_count_slots_and_stays_int32():
    from pyhgt_b200 import sampler
    dg = _Room()
    assert sampler._hit_capacity(dg, 1000) == 8000
    assert sampler._hit_capacity(dg, 0) == 0
    assert sampler._hit_capacity(dg, 2 ** 30) == 2 ** 31 - 1


def test_hit_room_grows_only_after_an_overflow():
    from pyhgt_b200 import sampler
    dg = _Room()
    sampler._grow_hit_room(dg, 8000, 1000)                # fitted exactly
    assert dg.hit_room == 8.0
    sampler._grow_hit_room(dg, 20000, 1000)               # did not fit: a quarter more than seen, per slot
    assert dg.hit_room == 25.0 and sampler._hit_capacity(dg, 1000) >= 20000
    sampler._grow_hit_room(dg, 100, 1000)                 # never shrinks
    assert dg.hit_room == 25.0
    sampler._grow_hit_room(dg, 5, 0)                      # no slots: nothing to learn
    assert dg.hit_room == 25.0


def test_host_entry_points_reject_bad_arguments():
    from pyhgt_b200 import _lib
    dptr = ctypes.c_void_p()
    with pytest.raises(_lib.HgtError, match="hgt_host_register"):
        _lib.call("hgt_host_register", None, 4096, ctypes.byref(dptr))
    buf = np.zeros(512, np.uint8)
    with pytest.raises(_lib.HgtError, match="hgt_host_register"):
        _lib.call("hgt_host_register", buf.ctypes.data, 0, ctypes.byref(dptr))
    with pytest.raises(_lib.HgtError, match="hgt_host_unregister"):
        _lib.call("hgt_host_unregister", None)
    st = ctypes.create_string_buffer(256)
    n = ctypes.c_int64()
    count = "hgt_gsample_batch_rebuild_count_host"
    with pytest.raises(_lib.HgtError, match=count):       # no hit counter
        _lib.call(count, None, None, 0, None, None, 0, 0, None, None, 0, None, None, None, None, None, 0, None)
    with pytest.raises(_lib.HgtError, match=count):       # records past 2^31 do not fit the int32 rank
        _lib.call(count, st, None, 0, None, None, 0, 0, None, buf.ctypes.data, 2 ** 31, ctypes.addressof(n), None,
                  None, None, None, 0, None)
    with pytest.raises(_lib.HgtError, match="hgt_gsample_batch_rebuild_write_host"):
        _lib.call("hgt_gsample_batch_rebuild_write_host", None, None, 0, None, None, None, None, None, None, None, 0,
                  None, 0, None, -1, None, 0, None, None, None, None, None, None, None)


def test_unpin_waits_out_a_stream_capture_and_keeps_buffers_cuda_refuses(monkeypatch):
    """The finalizer neither synchronises nor unregisters during a stream capture (that would invalidate the capture);
    the next call outside a capture unregisters every waiting buffer, each on its own, and keeps a buffer CUDA refused
    referenced so that its pages are not freed while registered."""
    from pyhgt_b200 import _lib, sampler
    calls, syncs = [], []
    capturing = [True]
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: capturing[0])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda dev=None: syncs.append(dev))
    bad = np.zeros(8, np.uint8)

    def fake_call(name, ptr):
        calls.append(ptr)
        if ptr == bad.ctypes.data:
            raise _lib.HgtError("refused")

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(sampler, "_UNPIN_LATER", [])
    monkeypatch.setattr(sampler, "_UNPIN_FAILED", [])
    a, b = np.zeros(8, np.uint8), np.zeros(8, np.uint8)
    sampler._unpin("cuda:0", [a, bad])
    assert calls == [] and syncs == [] and len(sampler._UNPIN_LATER) == 1
    capturing[0] = False
    sampler._unpin("cuda:1", [b])
    assert syncs == ["cuda:0", "cuda:1"]
    assert calls == [a.ctypes.data, bad.ctypes.data, b.ctypes.data]
    assert sampler._UNPIN_LATER == [] and len(sampler._UNPIN_FAILED) == 1 and sampler._UNPIN_FAILED[0] is bad
