"""CPU (-m "not gpu"): the split (phase 1 / phase 2) backward of lo_decoder_args in its generic mode, as the two-layer decoder of
the extension (latex_ocr_b200/ext.py TwoLayerDecoder) drives it.  dpred_ext is the generic-mode flag of both calls, so no field
was added; inconsistent phase / generic combinations are refused before any GPU work."""
import ctypes

import pytest

from latex_ocr_b200 import _lib


def _args(phase):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 2, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.phase = phase
    # never dereferenced: every case below is refused before any GPU work
    a.caps = a.enc = a.work = a.dlogits = 0x1000
    return a


@pytest.fixture
def lib_and_bt():
    L = _lib.lib()
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)
    return L, (ctypes.c_int32 * 3)(2, 2, 1)


def _call(L, a, bt, backward=True):
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    rc = L.lo_decoder_backward(ctypes.byref(a), None) if backward else L.lo_decoder_forward(ctypes.byref(a), 0, None)
    return rc, L.lo_last_error()


def test_generic_mode_is_flagged_by_dpred_ext_without_a_new_field():
    names = [f[0] for f in _lib.DecoderArgs._fields_]
    # the generic-mode fields keep their place: no field moved and none was appended after bfwork
    assert names[-2:] == ["work", "bfwork"]
    i = names.index("dalpha_ext")
    assert names[i:i + 3] == ["dalpha_ext", "dpred_ext", "dpred_stride"]
    assert names.index("phase") < names.index("bt_host")


def test_dalpha_ext_in_a_phase_2_backward_is_refused(lib_and_bt):
    L, bt = lib_and_bt
    a = _args(2)
    a.dpred_ext, a.dpred_stride, a.dalpha_ext = 0x1000, a.V, 0x1000
    rc, err = _call(L, a, bt)
    assert rc == -1 and b"phase 2 reads no d alpha" in err
    a = _args(2)                                             # also without the generic mode
    a.dalpha_ext = 0x1000
    rc, err = _call(L, a, bt)
    assert rc == -1 and b"phase 2 reads no d alpha" in err


@pytest.mark.parametrize("phase", [-1, 3])
@pytest.mark.parametrize("backward", [True, False])
def test_phase_outside_0_to_2_is_refused(lib_and_bt, phase, backward):
    L, bt = lib_and_bt
    rc, err = _call(L, _args(phase), bt, backward)
    assert rc == -1 and b"phase in 0..2" in err


def test_generic_phase_1_validates_dpred_ext(lib_and_bt):
    """dpred_ext, the mode flag, is checked in a phase-1 call too, although that call does not read it."""
    L, bt = lib_and_bt
    a = _args(1)
    a.dpred_ext, a.dpred_stride = 0x1000, a.V - 1
    rc, err = _call(L, a, bt)
    assert rc == -1 and b"dpred_stride >= V" in err
    a = _args(1)
    a.dpred_ext, a.dpred_stride, a.dlogits = 0x1000, a.V, None
    rc, err = _call(L, a, bt)
    assert rc == -1 and b"dpred_ext needs dlogits" in err
