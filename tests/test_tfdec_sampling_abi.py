"""CPU (-m "not gpu"): sampling on the TensorFlow-flavour decoder — the fields of lo_tfdec_args (fed, ss_prob, ss_u, ss_temp,
ss_gu, ss_state) are in the header-generated mirror after ``denc`` and before ``reg_off``, every inconsistent use of them and of the
TF-layout SCST entry points is refused before any GPU work, and tf_decoder.Decoder / img2seq_tf.Img2SeqModel check their
arguments."""
import ctypes
import math

import pytest

from latex_ocr_b200 import _lib, scst, tf_decoder

_FAKE = 0x1000          # never dereferenced: every call below is refused before any GPU work
_BUFFERS = ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init", "emb",
            "formula", "lengths", "loss", "denc", "g_w_img", "g_w_cat2", "g_beta", "g_w_lstm", "g_b_lstm", "g_w_oc", "g_w_y", "g_w_init",
            "g_b_init", "g_emb")
_SS = ("fed", "ss_prob", "ss_u", "ss_temp", "ss_gu", "ss_state")


@pytest.fixture
def L():
    return tf_decoder._bind()


def _args(**kw):
    """2 rows, T = 3, a consistent sampling block (fed, p, Philox state, tau); kw overrides (None clears a field)."""
    a = tf_decoder.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 2, 3, 8, 512, 256, 512, 512, 80, 40
    a.dt = _lib.LO_F32
    for k in _BUFFERS:
        setattr(a, k, _FAKE)
    a.formula_stride = a.T
    a.inv_n_words = 1.0
    a.fed = a.ss_prob = a.ss_state = a.ss_temp = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(L, a, entry):
    if entry == "forward":
        rc = L.lo_tfdec_forward(ctypes.byref(a), 0, None)
    elif entry == "backward":
        rc = L.lo_tfdec_backward(ctypes.byref(a), None)
    elif entry == "greedy":
        rc = L.lo_tfdec_greedy(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), None, None)
    elif entry == "beam":
        rc = L.lo_tfdec_beam(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                             ctypes.c_void_p(_FAKE), None)
    else:
        rc = L.lo_tfdec_beam_div(ctypes.byref(a), 1, 3, ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE), ctypes.c_void_p(_FAKE),
                                 ctypes.c_void_p(_FAKE), 1.0, 0.0, None, None, None)
    return rc, L.lo_last_error()


def test_sampling_fields_sit_between_denc_and_reg_off(L):
    names = [f[0] for f in tf_decoder.TfDecArgs._fields_]
    i = names.index("denc")
    assert tuple(names[i + 1:i + 7]) == _SS
    assert names[i + 7] == "reg_off"
    for n in _SS:
        assert dict(tf_decoder.TfDecArgs._fields_)[n] is ctypes.c_void_p, n
    assert names[-4:] == ["ws", "dlogits_ext", "dlogits_stride", "dalpha_ext"]
    assert L.lo_sizeof_tfdec_args() == ctypes.sizeof(tf_decoder.TfDecArgs)


@pytest.mark.parametrize("entry", ["forward", "backward"])
@pytest.mark.parametrize("kw, msg", [
    (dict(fed=None), b"needs fed"),
    (dict(ss_state=None), b"needs ss_u or ss_state"),
    (dict(ss_prob=None), b"need ss_prob"),                                   # ss_temp without ss_prob
    (dict(ss_prob=None, ss_temp=None, ss_gu=_FAKE), b"need ss_prob"),
    (dict(ss_temp=None, ss_gu=_FAKE), b"ss_gu (injected Gumbel uniforms) needs ss_temp"),
    (dict(rows_per_img=2), b"needs rows_per_img <= 1"),
])
def test_inconsistent_sampling_blocks_are_refused(L, entry, kw, msg):
    rc, err = _call(L, _args(**kw), entry)
    assert rc == -1 and msg in err, err


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_injected_coins_replace_the_philox_state(L, entry):
    """ss_u alone is a coin source: the coin check passes, and the check after it refuses the block"""
    rc, err = _call(L, _args(ss_state=None, ss_u=_FAKE, ss_temp=None, ss_gu=_FAKE), entry)
    assert rc == -1 and b"ss_gu (injected Gumbel uniforms) needs ss_temp" in err, err


@pytest.mark.parametrize("entry", ["greedy", "beam", "beam_div"])
@pytest.mark.parametrize("field", _SS)
def test_decode_entry_points_refuse_every_sampling_field(L, entry, field):
    kw = {k: None for k in _SS}
    kw[field] = _FAKE
    a = _args(**kw)
    a.rows_per_img = 1
    rc, err = _call(L, a, entry)
    assert rc == -1 and b"is a training mode" in err, err


def _reward_tf(L, **kw):
    p = dict(hyp=_FAKE, hs=4, Lh=4, greedy=_FAKE, gs=4, Lg=4, ref=_FAKE, rs=5, Lr=5, B=2, end=1, r_s=_FAKE, r_g=_FAKE, adv=_FAKE,
             n=_FAKE)
    p.update(kw)
    v = [None if x is None else (ctypes.c_void_p(x) if k in ("hyp", "greedy", "ref", "r_s", "r_g", "adv", "n") else x)
         for k, x in p.items()]
    return L.lo_scst_edit_reward_tf(*v, None), L.lo_last_error()


@pytest.mark.parametrize("kw, msg", [
    (dict(hyp=None), b"null pointer"), (dict(ref=None), b"null pointer"), (dict(r_s=None), b"null pointer"),
    (dict(B=0), b"B >= 1"), (dict(Lh=0), b"lengths in 1..512"), (dict(Lr=513, rs=513), b"lengths in 1..512"),
    (dict(Lg=0), b"greedy length"), (dict(hs=3), b"row strides"), (dict(gs=2), b"row strides"), (dict(rs=4), b"row strides"),
])
def test_edit_reward_tf_refusals(L, kw, msg):
    rc, err = _reward_tf(L, **kw)
    assert rc == -1 and msg in err


def _pg_tf(L, **kw):
    p = dict(logits=_FAKE, ldl=64, fed=_FAKE, fs=3, adv=_FAKE, n=_FAKE, temp=_FAKE, r_s=None, r_g=None, B=2, T=3, V=40, dpred=_FAKE,
             ds=40, partial=_FAKE, stats=_FAKE)
    p.update(kw)
    ptrs = ("logits", "fed", "adv", "n", "temp", "r_s", "r_g", "dpred", "partial", "stats")
    v = [ctypes.c_void_p(x) if (k in ptrs and x is not None) else x for k, x in p.items()]
    return L.lo_scst_pg_grad_tf(*v, None), L.lo_last_error()


@pytest.mark.parametrize("kw, msg", [
    (dict(logits=None), b"null pointer"), (dict(temp=None), b"null pointer"), (dict(n=None), b"null pointer"),
    (dict(partial=None), b"null pointer"), (dict(B=0), b"B, T >= 1"), (dict(T=70000, fs=70000), b"T <= 65535"),
    (dict(V=1, ldl=1, ds=1), b"V >= 2"), (dict(ldl=39), b"pred_stride"), (dict(ds=39), b"pred_stride"),
    (dict(fs=2), b"fed_stride >= T"),
])
def test_pg_grad_tf_refusals(L, kw, msg):
    rc, err = _pg_tf(L, **kw)
    assert rc == -1 and msg in err


def test_rewards_refuses_an_unknown_layout():
    with pytest.raises(ValueError, match="layout"):
        scst.rewards(None, None, 1, layout="batch")


@pytest.mark.parametrize("p, tau, msg", [(0.0, 0.5, "needs sampling_prob"), (1.0, -1.0, "sampling_temperature"),
                                         (1.0, math.nan, "sampling_temperature"), (1.0, math.inf, "sampling_temperature"),
                                         (-0.1, 0.0, "sampling_prob"), (1.5, 0.0, "sampling_prob")])
def test_decoder_checks_its_sampling_arguments_like_the_torch_flavour(p, tau, msg):
    from latex_ocr_b200.decoder import DecoderWithAttention
    with pytest.raises(ValueError, match=msg) as tf_err:
        tf_decoder.Decoder.check_sampling(p, tau)
    with pytest.raises(ValueError) as torch_err:
        DecoderWithAttention._forward_impl(object(), None, None, None, p, tau)
    assert str(tf_err.value) == str(torch_err.value)


class _Cfg:
    pass


def _model():
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    return Img2SeqModel(_Cfg(), device="cuda:0")      # constructing allocates nothing on the device


@pytest.mark.parametrize("p", [-0.1, 1.5, math.nan])
def test_set_sampling_prob_refuses_values_outside_0_1(p):
    m = _model()
    with pytest.raises(ValueError, match="sampling_prob"):
        m.set_sampling_prob(p)
    assert m.sampling_prob == 0.0


@pytest.mark.parametrize("tau", [-0.5, float("nan"), float("inf")])
def test_set_self_critical_refuses_bad_temperatures(tau):
    m = _model()
    with pytest.raises(ValueError, match="temperature"):
        m.set_self_critical(tau)
    assert m.scst_temperature == 0.0


def test_off_values_switch_back():
    m = _model()
    for tau in (None, 0, 0.0):
        m.set_self_critical(tau)
        assert m.scst_temperature == 0.0
    m.set_sampling_prob(0.3)
    m.set_sampling_prob(0)
    assert m.sampling_prob == 0.0


def test_self_critical_and_scheduled_sampling_exclude_each_other():
    m = _model()
    m.set_sampling_prob(0.25)
    with pytest.raises(_lib.LatexOcrB200Error, match="self-critical training and scheduled sampling exclude each other"):
        m.set_self_critical(1.0)
    m.set_sampling_prob(0.0)
    m.set_self_critical(1.0)
    with pytest.raises(_lib.LatexOcrB200Error, match="scheduled sampling and self-critical training exclude each other"):
        m.set_sampling_prob(0.5)
    assert m.sampling_prob == 0.0 and m.scst_temperature == 1.0


def test_self_critical_refuses_data_parallelism():
    m = _model()
    m.dist = object()
    with pytest.raises(_lib.LatexOcrB200Error, match="data parallelism"):
        m.set_self_critical(1.0)
    m.scst_temperature = 1.0              # as if set before dist was attached
    with pytest.raises(_lib.LatexOcrB200Error, match="data parallelism"):
        m.train_step(None, None)


def test_scheduled_sampling_keeps_data_parallelism():
    m = _model()
    m.dist = object()
    m.set_sampling_prob(0.5)
    assert m.sampling_prob == 0.5
