"""CPU (-m "not gpu"): the per-image region offsets (reg_off, reg_off_host) of both decoder flavours' argument blocks,
lo_decoder_args and lo_tfdec_args, are in the header-generated ctypes mirrors, and every inconsistent use is refused with LO_EINVAL
and the same messages before any GPU work.  Every call is parametrised by entry point: _greedy / _beam / forward / backward for the
torch flavour, the same with a tf prefix for the TensorFlow flavour."""
import ctypes

import pytest

from latex_ocr_b200 import _lib, tf_decoder

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000
_TF_BUFFERS = ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init",
               "emb", "formula", "lengths", "loss", "denc", "g_w_img", "g_w_cat2", "g_beta", "g_w_lstm", "g_b_lstm", "g_w_oc", "g_w_y",
               "g_w_init", "g_b_init", "g_emb")


@pytest.fixture
def L():
    return _lib.lib()


def _with(a, off, kw):
    """off: the host offsets (None: unset); kw: fields to set"""
    if off is not None:
        a._off = (ctypes.c_int32 * len(off))(*off)
        a.reg_off_host = ctypes.cast(a._off, ctypes.c_void_p)
        a.reg_off = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _args(off, **kw):
    """torch flavour: 3 images of at most R = 8 regions"""
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 3, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = _FAKE
    a._bt = (ctypes.c_int32 * 3)(3, 3, 3)
    a.bt_host = ctypes.cast(a._bt, ctypes.c_void_p)
    return _with(a, off, kw)


def _tf_args(off, **kw):
    """TF flavour: 3 images of at most R = 8 regions, one row each"""
    a = tf_decoder.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 3, 3, 8, 512, 256, 512, 512, 80, 40
    a.dt = _lib.LO_F32
    for k in _TF_BUFFERS:
        setattr(a, k, _FAKE)
    a.formula_stride = a.T
    a.inv_n_words = 1.0
    return _with(a, off, kw)


def _greedy(L, off, **kw):
    a = _args(off, **kw)
    rc = L.lo_decoder_greedy_hist(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), None, None)
    return rc, L.lo_last_error()


def _beam(L, off, **kw):
    a = _args(off, **dict({"rows_per_img": 1}, **kw))
    rc = L.lo_decoder_beam_div(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                               ctypes.c_void_p(_FAKE), 1.0, 0.0, None, None, None)
    return rc, L.lo_last_error()


def _tf_greedy(L, off, **kw):
    a = _tf_args(off, **kw)
    rc = L.lo_tfdec_greedy(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), None, None)
    return rc, L.lo_last_error()


def _tf_beam(L, off, **kw):
    a = _tf_args(off, **kw)
    rc = L.lo_tfdec_beam_div(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                             ctypes.c_void_p(_FAKE), 1.0, 0.0, None, None, None)
    return rc, L.lo_last_error()


DECODE = [_greedy, _beam, _tf_greedy, _tf_beam]
TRAIN = {"forward": (_args, lambda L, a: L.lo_decoder_forward(ctypes.byref(a), 0, None)),
         "backward": (_args, lambda L, a: L.lo_decoder_backward(ctypes.byref(a), None)),
         "tf_forward": (_tf_args, lambda L, a: L.lo_tfdec_forward(ctypes.byref(a), 0, None)),
         "tf_backward": (_tf_args, lambda L, a: L.lo_tfdec_backward(ctypes.byref(a), None))}


def test_region_offset_fields_are_pointers_in_the_mirror(L):
    """adjacent in both mirrors; in lo_tfdec_args right before ``ws``"""
    for mirror, sizeof, after in ((_lib.DecoderArgs, L.lo_sizeof_decoder_args, "work"),
                                  (tf_decoder.TfDecArgs, L.lo_sizeof_tfdec_args, "ws")):
        fields = dict(mirror._fields_)
        names = [f[0] for f in mirror._fields_]
        assert fields["reg_off"] is ctypes.c_void_p and fields["reg_off_host"] is ctypes.c_void_p
        assert names.index("reg_off") + 1 == names.index("reg_off_host") < names.index(after)
        assert sizeof() == ctypes.sizeof(mirror)
    names = [f[0] for f in tf_decoder.TfDecArgs._fields_]
    assert names.index("reg_off_host") == names.index("ws") - 1


@pytest.mark.parametrize("entry", list(TRAIN))
def test_offsets_on_the_training_entry_points_are_refused(L, entry):
    args, call = TRAIN[entry]
    for kw in ({}, {"reg_off": None}):
        rc = call(L, args([0, 2, 5, 8], **kw))
        assert rc == -1 and b"decode entry points only" in L.lo_last_error()


@pytest.mark.parametrize("call", DECODE)
def test_one_field_without_the_other_is_refused(L, call):
    rc, err = call(L, [0, 2, 5, 8], reg_off=None)
    assert rc == -1 and b"set together" in err
    rc, err = call(L, None, reg_off=_FAKE)
    assert rc == -1 and b"set together" in err


@pytest.mark.parametrize("call", DECODE)
def test_offsets_must_start_at_zero(L, call):
    rc, err = call(L, [1, 3, 5, 8])
    assert rc == -1 and b"reg_off_host[0] must be 0" in err


@pytest.mark.parametrize("call", DECODE)
@pytest.mark.parametrize("off", [[0, 2, 2, 8], [0, 3, 1, 4], [0, 9, 12, 14], [0, 1, 2, 11]])
def test_region_counts_outside_one_to_R_are_refused(L, call, off):
    rc, err = call(L, off)
    assert rc == -1 and b"region count of every image in 1..R" in err


def test_beam_rows_share_their_image_offsets(L):
    """rows_per_img = 3: one image of 3 rows, so only reg_off_host[0..1] are read; a count above R is still refused (both
    flavours' beam entry points)"""
    for call in (_beam, _tf_beam):
        rc, err = call(L, [0, 9], rows_per_img=3)
        assert rc == -1 and b"region count of every image in 1..R" in err, call.__name__


@pytest.mark.parametrize("call", DECODE)
def test_offsets_need_the_pipelined_attention_kernels(L, call):
    with _lib.option(att_pipe=0):
        rc, err = call(L, [0, 2, 5, 8])
    assert rc == -1 and b"att_pipe = 1" in err
