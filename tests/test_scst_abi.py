"""CPU (-m "not gpu"): self-critical training's ABI — the sampling-temperature fields of lo_decoder_args (ss_temp, ss_gu) are in the
header-generated mirror, every inconsistent use of them and of lo_scst_edit_reward / lo_scst_pg_grad is refused before any GPU work,
the Gumbel uniforms' Philox counters are disjoint from the dropout and coin streams, and the Python entry points check their
arguments."""
import ctypes
import math

import numpy as np
import pytest

from latex_ocr_b200 import _lib, philox

_FAKE = 0x1000          # never dereferenced: every call below is refused before any GPU work


def _args(**kw):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 2, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = a.dlogits = _FAKE
    a.fed = a.ss_prob = a.dropout_state = a.ss_temp = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.fixture
def L():
    return _lib.lib()


def _call(L, a, entry):
    bt = (ctypes.c_int32 * 3)(2, 2, 2)
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    if entry == "forward":
        rc = L.lo_decoder_forward(ctypes.byref(a), 0, None)
    elif entry == "backward":
        rc = L.lo_decoder_backward(ctypes.byref(a), None)
    elif entry == "greedy":
        rc = L.lo_decoder_greedy(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), None)
    else:
        a.rows_per_img = 1
        rc = L.lo_decoder_beam(ctypes.byref(a), 0, 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                               ctypes.c_void_p(_FAKE), None)
    return rc, L.lo_last_error()


def test_temperature_fields_follow_the_sampling_block(L):
    names = [f[0] for f in _lib.DecoderArgs._fields_]
    i = names.index("ss_u")
    assert names[i + 1:i + 3] == ["ss_temp", "ss_gu"]
    for n in ("ss_temp", "ss_gu"):
        assert dict(_lib.DecoderArgs._fields_)[n] is ctypes.c_void_p
    assert names[-2:] == ["work", "bfwork"]
    assert L.lo_sizeof_decoder_args() == ctypes.sizeof(_lib.DecoderArgs)


@pytest.mark.parametrize("entry", ["forward", "backward", "greedy", "beam"])
@pytest.mark.parametrize("field", ["ss_temp", "ss_gu"])
def test_temperature_fields_without_ss_prob_are_refused(L, entry, field):
    kw = {"ss_prob": None, "ss_temp": None, field: _FAKE}
    rc, err = _call(L, _args(**kw), entry)
    assert rc == -1 and b"need ss_prob" in err


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_injected_gumbel_uniforms_without_ss_temp_are_refused(L, entry):
    rc, err = _call(L, _args(ss_temp=None, ss_gu=_FAKE), entry)
    assert rc == -1 and b"ss_gu (injected Gumbel uniforms) needs ss_temp" in err


def test_greedy_and_beam_still_refuse_ss_prob_with_a_temperature(L):
    rc, err = _call(L, _args(), "greedy")
    assert rc == -1 and b"greedy decode" in err
    rc, err = _call(L, _args(), "beam")
    assert rc == -1 and b"beam search" in err


def _reward(L, **kw):
    p = dict(hyp=_FAKE, hs=4, Lh=4, greedy=_FAKE, gs=4, Lg=4, ref=_FAKE, rs=5, Lr=5, B=2, end=1, r_s=_FAKE, r_g=_FAKE, adv=_FAKE,
             n=_FAKE)
    p.update(kw)
    v = [None if x is None else (ctypes.c_void_p(x) if k in ("hyp", "greedy", "ref", "r_s", "r_g", "adv", "n") else x)
         for k, x in p.items()]
    return L.lo_scst_edit_reward(*v, None), L.lo_last_error()


@pytest.mark.parametrize("kw, msg", [
    (dict(hyp=None), b"null pointer"), (dict(ref=None), b"null pointer"), (dict(r_s=None), b"null pointer"),
    (dict(B=0), b"B >= 1"), (dict(Lh=0), b"lengths in 1..512"), (dict(Lr=513, rs=513), b"lengths in 1..512"),
    (dict(Lg=0), b"greedy length"), (dict(hs=3), b"row strides"), (dict(gs=2), b"row strides"), (dict(rs=4), b"row strides"),
])
def test_edit_reward_refusals(L, kw, msg):
    rc, err = _reward(L, **kw)
    assert rc == -1 and msg in err


def _pg(L, **kw):
    p = dict(preds=_FAKE, ps=40, fed=_FAKE, fs=3, adv=_FAKE, n=_FAKE, temp=_FAKE, r_s=None, r_g=None, B=2, T=3, V=40, dpred=_FAKE,
             ds=40, partial=_FAKE, stats=_FAKE)
    p.update(kw)
    ptrs = ("preds", "fed", "adv", "n", "temp", "r_s", "r_g", "dpred", "partial", "stats")
    v = [ctypes.c_void_p(x) if (k in ptrs and x is not None) else x for k, x in p.items()]
    return L.lo_scst_pg_grad(*v, None), L.lo_last_error()


@pytest.mark.parametrize("kw, msg", [
    (dict(preds=None), b"null pointer"), (dict(temp=None), b"null pointer"), (dict(n=None), b"null pointer"),
    (dict(partial=None), b"null pointer"), (dict(B=0), b"B, T >= 1"), (dict(V=1, ps=1, ds=1), b"V >= 2"),
    (dict(ps=39), b"pred_stride"), (dict(ds=39), b"pred_stride"), (dict(fs=2), b"fed_stride >= T"),
])
def test_pg_grad_refusals(L, kw, msg):
    rc, err = _pg(L, **kw)
    assert rc == -1 and msg in err


def test_gumbel_mirror_is_the_documented_philox_draw():
    seed, call, B, T, V = 0x0123456789ABCDEF, 5, 3, 4, 13
    u = philox.gumbel_uniforms(seed, call, B, T, V)
    assert u.shape == (B, T, V) and u.dtype == np.float64
    assert (u > 0).all() and (u < 1).all()
    for b in range(B):
        for t in range(T):
            for v in range(V):
                w = philox.philox4x32_10(0x80000000 | (v >> 2), t, b, call, seed & 0xFFFFFFFF, seed >> 32)
                assert u[b, t, v] == ((int(w[v & 3]) >> 8) + 0.5) * 2.0 ** -24
    assert not np.array_equal(u, philox.gumbel_uniforms(seed, call + 1, B, T, V))
    # the extremes of the word map to (0, 1) open at both ends
    assert ((0 >> 8) + 0.5) * 2.0 ** -24 > 0 and (((2 ** 32 - 1) >> 8) + 0.5) * 2.0 ** -24 < 1


def test_gumbel_counters_are_disjoint_from_the_dropout_and_coin_streams():
    """First counter words over the full index ranges (a unit j or token v is a non-negative int32): dropout j >> 2 lies in
    [0, 2^29), the coin is 0xFFFFFFFF, the Gumbel uniforms 0x80000000 | v >> 2 lie in [2^31, 2^31 + 2^29).  The other three words
    (t, b, call) are shared, so the streams never meet."""
    idx_max = 2 ** 31 - 1
    dropout = (0, idx_max >> 2)
    gumbel = (0x80000000 | 0, 0x80000000 | (idx_max >> 2))
    coin = 0xFFFFFFFF
    assert dropout[1] < gumbel[0] and gumbel[1] < coin
    # and the mirrors draw from those words: at a practical size no Gumbel word equals a dropout or coin word of the same (b, t, call)
    seed, call, B, T, D, V = 11, 2, 3, 4, 512, 500
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    t = np.arange(T, dtype=np.uint64)[None, :, None]
    j4 = np.arange(D // 4, dtype=np.uint64)[None, None, :]
    v4 = np.arange(V // 4, dtype=np.uint64)[None, None, :]
    drop = np.stack(philox.philox4x32_10(j4 + 0 * b + 0 * t, t + 0 * b + 0 * j4, b + 0 * t + 0 * j4, np.uint64(call), seed, 0), -1)
    gum = np.stack(philox.philox4x32_10(np.uint64(0x80000000) | (v4 + 0 * b + 0 * t), t + 0 * b + 0 * v4, b + 0 * t + 0 * v4,
                                        np.uint64(call), seed, 0), -1)
    coinw = philox.philox4x32_10(np.uint64(0xFFFFFFFF) + 0 * b + 0 * t, t + 0 * b, b + 0 * t, np.uint64(call), seed, 0)[0]
    assert not np.isin(gum, drop).any()
    assert not np.isin(gum, coinw).any()
    u = philox.gumbel_uniforms(seed, call, B, T, V)
    assert np.array_equal(u, ((gum.reshape(B, T, V) >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24)


class _Cfg:
    pass


def _model():
    from latex_ocr_b200.img2seq import Img2SeqModel
    return Img2SeqModel(_Cfg(), n_tok=40, device="cuda:0")      # constructing allocates nothing on the device


@pytest.mark.parametrize("tau", [-0.5, float("nan"), float("inf")])
def test_set_self_critical_refuses_bad_temperatures(tau):
    m = _model()
    with pytest.raises(ValueError, match="temperature"):
        m.set_self_critical(tau)
    assert m.scst_temperature == 0.0


def test_set_self_critical_off_values_are_cross_entropy():
    m = _model()
    for tau in (None, 0, 0.0):
        m.set_self_critical(tau)
        assert m.scst_temperature == 0.0


def test_self_critical_and_scheduled_sampling_exclude_each_other():
    m = _model()
    m.sampling_prob = 0.25
    with pytest.raises(_lib.LatexOcrB200Error, match="scheduled sampling"):
        m.set_self_critical(1.0)
    m.sampling_prob = 0.0
    m.scst_temperature = 1.0              # as set_self_critical(1.0) leaves it (which would allocate tau on the device)
    with pytest.raises(_lib.LatexOcrB200Error, match="self-critical"):
        m.set_sampling_prob(0.5)
    m.set_sampling_prob(0.0)


def test_self_critical_refuses_data_parallelism():
    import torch
    m = _model()
    m.dist = object()
    with pytest.raises(_lib.LatexOcrB200Error, match="data parallelism"):
        m.set_self_critical(1.0)
    m.scst_temperature = 1.0
    with pytest.raises(_lib.LatexOcrB200Error, match="data parallelism"):
        m.train_step(torch.zeros(2, 1, 8, 8), torch.zeros(2, 4, dtype=torch.int64))


def test_the_two_layer_extension_refuses_self_critical_training():
    from latex_ocr_b200.ext import Img2SeqRowModel
    with pytest.raises(_lib.LatexOcrB200Error, match="self-critical"):
        Img2SeqRowModel.set_self_critical(None, 1.0)
    Img2SeqRowModel.set_self_critical(None, None)


@pytest.mark.parametrize("p, tau, msg", [(0.0, 0.5, "needs sampling_prob"), (1.0, -1.0, "sampling_temperature"),
                                         (1.0, math.nan, "sampling_temperature")])
def test_decoder_forward_checks_the_temperature_first(p, tau, msg):
    from latex_ocr_b200.decoder import DecoderWithAttention
    with pytest.raises(ValueError, match=msg):
        DecoderWithAttention._forward_impl(object(), None, None, None, p, tau)
