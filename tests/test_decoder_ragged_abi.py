"""CPU (-m "not gpu"): the per-image region offsets of lo_decoder_args (reg_off, reg_off_host) are in the header-generated ctypes
mirror, and every inconsistent use is refused with LO_EINVAL before any GPU work."""
import ctypes

import pytest

from latex_ocr_b200 import _lib

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000


@pytest.fixture
def L():
    return _lib.lib()


def _args(off, **kw):
    """3 images of at most R = 8 regions, beam rows_per_img; off: the host offsets (None: unset)."""
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 3, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = _FAKE
    a._bt = (ctypes.c_int32 * 3)(3, 3, 3)
    a.bt_host = ctypes.cast(a._bt, ctypes.c_void_p)
    if off is not None:
        a._off = (ctypes.c_int32 * len(off))(*off)
        a.reg_off_host = ctypes.cast(a._off, ctypes.c_void_p)
        a.reg_off = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _greedy(L, a):
    rc = L.lo_decoder_greedy_hist(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), None, None)
    return rc, L.lo_last_error()


def _beam(L, a):
    a.rows_per_img = 1
    rc = L.lo_decoder_beam_div(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                               ctypes.c_void_p(_FAKE), 1.0, 0.0, None, None, None)
    return rc, L.lo_last_error()


def test_region_offset_fields_are_pointers_in_the_mirror(L):
    fields = dict(_lib.DecoderArgs._fields_)
    names = [f[0] for f in _lib.DecoderArgs._fields_]
    assert fields["reg_off"] is ctypes.c_void_p and fields["reg_off_host"] is ctypes.c_void_p
    assert names.index("reg_off") + 1 == names.index("reg_off_host") < names.index("work")
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_offsets_on_the_training_entry_points_are_refused(L, entry):
    for kw in ({}, {"reg_off": None}):
        a = _args([0, 2, 5, 8], **kw)
        rc = L.lo_decoder_forward(ctypes.byref(a), 0, None) if entry == "forward" else L.lo_decoder_backward(ctypes.byref(a), None)
        assert rc == -1 and b"decode entry points only" in L.lo_last_error()


@pytest.mark.parametrize("call", [_greedy, _beam])
def test_one_field_without_the_other_is_refused(L, call):
    rc, err = call(L, _args([0, 2, 5, 8], reg_off=None))
    assert rc == -1 and b"set together" in err
    rc, err = call(L, _args(None, reg_off=_FAKE))
    assert rc == -1 and b"set together" in err


@pytest.mark.parametrize("call", [_greedy, _beam])
def test_offsets_must_start_at_zero(L, call):
    rc, err = call(L, _args([1, 3, 5, 8]))
    assert rc == -1 and b"reg_off_host[0] must be 0" in err


@pytest.mark.parametrize("call", [_greedy, _beam])
@pytest.mark.parametrize("off", [[0, 2, 2, 8], [0, 3, 1, 4], [0, 9, 12, 14], [0, 1, 2, 11]])
def test_region_counts_outside_one_to_R_are_refused(L, call, off):
    rc, err = call(L, _args(off))
    assert rc == -1 and b"region count of every image in 1..R" in err


@pytest.mark.parametrize("call", [_greedy, _beam])
def test_offsets_need_the_pipelined_attention_kernels(L, call):
    with _lib.option(att_pipe=0):
        rc, err = call(L, _args([0, 2, 5, 8]))
    assert rc == -1 and b"att_pipe = 1" in err
