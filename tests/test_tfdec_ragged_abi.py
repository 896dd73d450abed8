"""CPU (-m "not gpu"): the per-image region offsets of lo_tfdec_args (reg_off, reg_off_host) are in the header-generated ctypes
mirror before ``ws``, and every inconsistent use is refused with LO_EINVAL and the torch flavour's messages before any GPU work."""
import ctypes

import pytest

from latex_ocr_b200 import _lib, tf_decoder

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000
_BUFFERS = ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init", "emb",
            "formula", "lengths", "loss", "denc", "g_w_img", "g_w_cat2", "g_beta", "g_w_lstm", "g_b_lstm", "g_w_oc", "g_w_y", "g_w_init",
            "g_b_init", "g_emb")


@pytest.fixture
def L():
    return tf_decoder._bind()


def _args(off, **kw):
    """3 images of at most R = 8 regions, one row each; off: the host offsets (None: unset)."""
    a = tf_decoder.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 3, 3, 8, 512, 256, 512, 512, 80, 40
    a.dt = _lib.LO_F32
    for k in _BUFFERS:
        setattr(a, k, _FAKE)
    a.formula_stride = a.T
    a.inv_n_words = 1.0
    if off is not None:
        a._off = (ctypes.c_int32 * len(off))(*off)
        a.reg_off_host = ctypes.cast(a._off, ctypes.c_void_p)
        a.reg_off = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _greedy(L, a):
    rc = L.lo_tfdec_greedy(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), None, None)
    return rc, L.lo_last_error()


def _beam(L, a):
    rc = L.lo_tfdec_beam_div(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                             ctypes.c_void_p(_FAKE), 1.0, 0.0, None, None, None)
    return rc, L.lo_last_error()


def test_region_offset_fields_are_adjacent_pointers_before_ws(L):
    fields = dict(tf_decoder.TfDecArgs._fields_)
    names = [f[0] for f in tf_decoder.TfDecArgs._fields_]
    assert fields["reg_off"] is ctypes.c_void_p and fields["reg_off_host"] is ctypes.c_void_p
    assert names.index("reg_off") + 1 == names.index("reg_off_host") == names.index("ws") - 1
    assert L.lo_sizeof_tfdec_args() == ctypes.sizeof(tf_decoder.TfDecArgs)


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_offsets_on_the_training_entry_points_are_refused(L, entry):
    for kw in ({}, {"reg_off": None}):
        a = _args([0, 2, 5, 8], **kw)
        rc = L.lo_tfdec_forward(ctypes.byref(a), 0, None) if entry == "forward" else L.lo_tfdec_backward(ctypes.byref(a), None)
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


def test_beam_rows_share_their_image_offsets(L):
    """rows_per_img = 3: one image of 3 rows, so only reg_off_host[0..1] are read; a count above R is still refused"""
    rc, err = _beam(L, _args([0, 9], rows_per_img=3))
    assert rc == -1 and b"region count of every image in 1..R" in err


@pytest.mark.parametrize("call", [_greedy, _beam])
def test_offsets_need_the_pipelined_attention_kernels(L, call):
    with _lib.option(att_pipe=0):
        rc, err = call(L, _args([0, 2, 5, 8]))
    assert rc == -1 and b"att_pipe = 1" in err
