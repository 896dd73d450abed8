"""CPU (-m "not gpu"): the scheduled-sampling fields of lo_decoder_args (fed, ss_prob, ss_u) are in the header-generated ctypes
mirror, every inconsistent use is refused before any GPU work, and the host mirror of the sampling coin is the documented Philox
draw, disjoint from the dropout stream."""
import ctypes

import numpy as np
import pytest

from latex_ocr_b200 import _lib, philox

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000


def _args(**kw):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 2, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = a.dlogits = _FAKE
    a.fed = a.ss_prob = a.dropout_state = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.fixture
def L():
    return _lib.lib()


def _bt():
    return (ctypes.c_int32 * 3)(2, 2, 1)


def _forward(L, a):
    bt = _bt()
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    return L.lo_decoder_forward(ctypes.byref(a), 0, None), L.lo_last_error()


def _backward(L, a):
    bt = _bt()
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    return L.lo_decoder_backward(ctypes.byref(a), None), L.lo_last_error()


def test_sampling_fields_are_in_the_mirror_before_work(L):
    names = [f[0] for f in _lib.DecoderArgs._fields_]
    i = names.index("caps_stride")
    assert names[i + 1:i + 4] == ["fed", "ss_prob", "ss_u"]
    for n in ("fed", "ss_prob", "ss_u"):
        assert dict(_lib.DecoderArgs._fields_)[n] is ctypes.c_void_p
    # the layout the other ABI tests pin is unchanged
    assert names[-2:] == ["work", "bfwork"]
    assert names.index("phase") < names.index("bt_host")
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)


@pytest.mark.parametrize("call", [_forward, _backward])
def test_ss_prob_without_fed_is_refused(L, call):
    rc, err = call(L, _args(fed=None))
    assert rc == -1 and b"needs fed" in err


@pytest.mark.parametrize("call", [_forward, _backward])
def test_ss_prob_without_a_coin_source_is_refused(L, call):
    rc, err = call(L, _args(dropout_state=None, ss_u=None))
    assert rc == -1 and b"needs ss_u or dropout_state" in err
    # an injected coin alone is enough to pass this check (the call then fails later, on the fake phase below)
    rc, err = call(L, _args(dropout_state=None, ss_u=_FAKE, phase=1))
    assert rc == -1 and b"needs phase 0" in err


@pytest.mark.parametrize("phase", [1, 2])
@pytest.mark.parametrize("call", [_forward, _backward])
def test_ss_prob_with_a_phase_is_refused(L, call, phase):
    rc, err = call(L, _args(phase=phase))
    assert rc == -1 and b"needs phase 0" in err


def test_ss_prob_with_rows_per_img_is_refused(L):
    rc, err = _forward(L, _args(rows_per_img=2))
    assert rc == -1 and b"rows_per_img <= 1" in err


def test_ss_prob_on_the_decode_entry_points_is_refused(L):
    bt = (ctypes.c_int32 * 3)(2, 2, 2)
    a = _args()
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    rc = L.lo_decoder_greedy(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), None)
    assert rc == -1 and b"greedy decode" in L.lo_last_error()
    rc = L.lo_decoder_greedy_hist(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), None, None)
    assert rc == -1 and b"greedy decode" in L.lo_last_error()
    a.rows_per_img = 1
    rc = L.lo_decoder_beam(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                           ctypes.c_void_p(_FAKE), None)
    assert rc == -1 and b"beam search" in L.lo_last_error()


def test_sampling_coin_mirror_is_the_documented_philox_draw():
    seed, call, B, T = 0x0123456789ABCDEF, 7, 5, 9
    u = philox.sampling_uniforms(seed, call, B, T)
    assert u.shape == (B, T) and u.dtype == np.float32
    assert (u >= 0).all() and (u < 1).all()
    for b in range(B):
        for t in range(T):
            w = philox.philox4x32_10(0xFFFFFFFF, t, b, call, seed & 0xFFFFFFFF, seed >> 32)
            assert u[b, t] == np.float32(int(w[0]) >> 8) * np.float32(2.0 ** -24)
    # another call counter or seed draws other coins
    assert not np.array_equal(u, philox.sampling_uniforms(seed, call + 1, B, T))
    assert not np.array_equal(u, philox.sampling_uniforms(seed + 1, call, B, T))


def test_sampling_coins_differ_from_the_dropout_stream():
    """The coin's first counter word (0xFFFFFFFF) is one the dropout stream (j >> 2 < D / 4) never uses: no coin equals the
    dropout uniform of the same (row, step, call)."""
    seed, call, B, T, D = 99, 3, 4, 6, 512
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    t = np.arange(T, dtype=np.uint64)[None, :, None]
    j4 = np.arange(D // 4, dtype=np.uint64)[None, None, :]
    coin = philox.philox4x32_10(np.uint64(0xFFFFFFFF) + 0 * b + 0 * t, t + 0 * b, b + 0 * t, np.uint64(call), seed, 0)[0]
    drop = np.stack(philox.philox4x32_10(j4 + 0 * b + 0 * t, t + 0 * b + 0 * j4, b + 0 * t + 0 * j4, np.uint64(call), seed, 0), -1)
    assert drop.shape == (B, T, D // 4, 4)
    assert not (drop == coin[:, :, :, None]).any()
    # and the mirror's coins are those words
    assert np.array_equal(philox.sampling_uniforms(seed, call, B, T), philox.u01(coin).reshape(B, T))


def test_the_two_layer_extension_refuses_sampling():
    """The second decoder layer sits between the cell and fc: no per-step prediction to feed back, refused before any work."""
    import torch.nn as nn
    from latex_ocr_b200.ext import Img2SeqRowModel, TwoLayerDecoder
    with pytest.raises(_lib.LatexOcrB200Error, match="scheduled sampling"):
        TwoLayerDecoder(nn.Identity(), nn.Identity())(None, None, None, sampling_prob=0.5)
    with pytest.raises(_lib.LatexOcrB200Error, match="scheduled sampling"):
        Img2SeqRowModel.set_sampling_prob(None, 0.5)
    Img2SeqRowModel.set_sampling_prob(None, 0.0)          # p = 0 is teacher forcing: accepted
