"""CPU (-m "not gpu"): the generic-mode fields of lo_decoder_args (upstream gradient of the predictions) are in the ctypes
mirror, and lo_decoder_backward validates them before it touches the device."""
import ctypes

from latex_ocr_b200 import _lib


def test_generic_backward_fields_and_validation_without_gpu():
    L = _lib.lib()
    names = [f[0] for f in _lib.DecoderArgs._fields_]
    assert "dpred_ext" in names and "dpred_stride" in names
    assert dict(_lib.DecoderArgs._fields_)["dpred_stride"] is ctypes.c_int64
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 2, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    bt = (ctypes.c_int32 * 3)(2, 2, 1)
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    # never dereferenced: the arguments are refused before any GPU work
    a.caps = a.enc = a.work = a.dlogits = a.dpred_ext = 0x1000
    a.dpred_stride = a.V - 1
    assert L.lo_decoder_backward(ctypes.byref(a), None) == -1
    assert b"dpred_stride >= V" in L.lo_last_error()
    a.dpred_stride, a.dlogits = a.V, None
    assert L.lo_decoder_backward(ctypes.byref(a), None) == -1
    assert b"dpred_ext needs dlogits" in L.lo_last_error()
