"""CPU (-m "not gpu"): greedy and beam decode of the two-layer decoder (lo_decoder2_greedy / lo_decoder2_beam).  The layer struct
and both entry points are bound from the header; every bad call is refused with LO_EINVAL before any GPU work; and the CPU oracle
of tests/decoder2_decode_oracle.py is consistent with oracle/ref_ext.py: the logits along its greedy path are decoder2_forward
teacher-forced on those tokens, and its beam search of width 1 chooses the greedy tokens."""
import ctypes

import pytest
import torch

import decoder2_decode_oracle as d2o
from latex_ocr_b200 import _lib

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000


@pytest.fixture
def L():
    return _lib.lib()


def _args(beam=1, off=None, **kw):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 3 * beam, 3, 8, 512, 512, 512, 512, 40
    a.rows_per_img = beam
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = a.row_loss = _FAKE
    a._bt = (ctypes.c_int32 * 3)(3 * beam, 3 * beam, 3 * beam)
    a.bt_host = ctypes.cast(a._bt, ctypes.c_void_p)
    if off is not None:
        a._off = (ctypes.c_int32 * len(off))(*off)
        a.reg_off_host = ctypes.cast(a._off, ctypes.c_void_p)
        a.reg_off = _FAKE
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _layer(**kw):
    l2 = _lib.Decoder2Layer()
    l2.w_ih = l2.w_hh = l2.b_ih = l2.b_hh = l2.scratch = _FAKE
    for k, v in kw.items():
        setattr(l2, k, v)
    return l2


def _greedy(L, a, l2, max_steps=3):
    o = [ctypes.c_void_p(_FAKE)] * 3
    rc = L.lo_decoder2_greedy(ctypes.byref(a), l2, 0, 1, max_steps, *o, None)
    return rc, L.lo_last_error()


def _beam(L, a, l2, pen=None, max_steps=3, div=(1.0, 0.0, None, None)):
    o = [ctypes.c_void_p(_FAKE)] * 4
    rc = L.lo_decoder2_beam(ctypes.byref(a), l2, 0, 1, max_steps, *o, *div, pen, None)
    return rc, L.lo_last_error()


def test_bound_from_the_header(L):
    sigs = _lib.declared_signatures()
    assert [f[0] for f in _lib.Decoder2Layer._fields_] == ["w_ih", "w_hh", "b_ih", "b_hh", "scratch"]
    assert L.lo_sizeof_decoder2_layer() == ctypes.sizeof(_lib.Decoder2Layer)
    layer = ctypes.POINTER(_lib.Decoder2Layer)
    # the torch flavour's entry point with the layer after the args
    for name, base in (("lo_decoder2_greedy", "lo_decoder_greedy_hist"), ("lo_decoder2_beam", "lo_decoder_beam_pen")):
        restype, argtypes = sigs[name]
        want = list(sigs[base][1])
        assert restype is ctypes.c_int and argtypes == want[:1] + [layer] + want[1:], name
        assert getattr(L, name).argtypes == argtypes
    assert sigs["lo_decoder2_scratch_bytes"] == (ctypes.c_int64, [ctypes.POINTER(_lib.DecoderArgs)])


def test_scratch_bytes(L):
    """two slots of h2, c2 (fp32) and of the bf16 mirror of h2, the [B][4D] gates and the summed bias, each 256-byte aligned"""
    a = _args()
    for B, D in ((3, 512), (1280, 512), (7, 64)):
        a.B, a.D = B, D
        want = sum((x + 255) // 256 * 256 for x in (16 * B * D, 8 * B * D, 8 * B * D, 4 * B * D, 16 * D))
        assert L.lo_decoder2_scratch_bytes(ctypes.byref(a)) == want
    assert L.lo_decoder2_scratch_bytes(None) == 0


BAD = [
    ("null layer", dict(layer=None), b"null lo_decoder2_layer"),
    ("null w_ih", dict(w_ih=None), b"null layer-2 weight"),
    ("null w_hh", dict(w_hh=None), b"null layer-2 weight"),
    ("null b_ih", dict(b_ih=None), b"null layer-2 weight"),
    ("null b_hh", dict(b_hh=None), b"null layer-2 weight"),
    ("null scratch", dict(scratch=None), b"null layer-2 weight"),
    ("phase 1", dict(phase=1), b"phase must be 0"),
    ("phase 2", dict(phase=2), b"phase must be 0"),
    ("scheduled sampling", dict(ss_prob=_FAKE, fed=_FAKE, ss_u=_FAKE), b"scheduled sampling"),
    ("null args", dict(args=None), b"null args"),
    ("bad region offsets", dict(off=[1, 3, 5, 8]), b"reg_off_host[0] must be 0"),
    ("max_steps above T", dict(max_steps=4), b"max_steps"),
    ("null enc", dict(enc=None), b"null pointer"),
]


def _split(kw):
    kw = dict(kw)
    layer = {k: kw.pop(k) for k in ("w_ih", "w_hh", "b_ih", "b_hh", "scratch") if k in kw}
    l2 = None if "layer" in kw and kw.pop("layer") is None else ctypes.byref(_layer(**layer))
    return kw.pop("max_steps", 3), kw.pop("off", None), kw.pop("args", True), l2, kw


@pytest.mark.parametrize("entry", ["greedy", "beam"])
@pytest.mark.parametrize("what,kw,msg", BAD, ids=[b[0] for b in BAD])
def test_bad_calls_are_refused(L, entry, what, kw, msg):
    max_steps, off, has_args, l2, akw = _split(kw)
    beam = 1 if entry == "greedy" else 2
    a = _args(beam, off, **akw)
    if not has_args:
        fn = L.lo_decoder2_greedy if entry == "greedy" else L.lo_decoder2_beam
        o = [ctypes.c_void_p(_FAKE)] * (3 if entry == "greedy" else 4)
        rest = () if entry == "greedy" else (1.0, 0.0, None, None, None)
        rc, err = fn(None, l2, 0, 1, 3, *o, *rest, None), L.lo_last_error()
    elif entry == "greedy":
        rc, err = _greedy(L, a, l2, max_steps)
    else:
        rc, err = _beam(L, a, l2, max_steps=max_steps)
    assert rc == -1 and msg in err, err


def _penalty(**kw):
    p = _lib.BeamPenalty()
    p.alpha, p.beta = 0.6, 0.2
    p.len_pen = p.cov = p.len = p.scores = _FAKE
    for k, v in kw.items():
        setattr(p, k, v)
    return p


BEAM_BAD = [
    ("alpha < 0", dict(pen=dict(alpha=-0.1)), b"finite and >= 0"),
    ("alpha without len_pen", dict(pen=dict(len_pen=None)), b"needs the len_pen table"),
    ("beta without cov", dict(pen=dict(cov=None)), b"needs the cov scratch"),
    ("null len", dict(pen=dict(len=None)), b"null len scratch"),
    ("diversity without a source", dict(div=(0.5, 0.7, None, None)), b"diversity penalty needs"),
    ("beam above 16", dict(beam=17), b"1 <= beam"),
    ("beam above V", dict(beam=4, V=3), b"beam (rows_per_img) <= V"),
    ("beam above V with a penalty", dict(beam=16, V=15, pen={}), b"beam (rows_per_img) <= V"),
    ("beam*V too large", dict(beam=16, V=2000, pen={}), b"beam*V too large"),
]


@pytest.mark.parametrize("what,kw,msg", BEAM_BAD, ids=[b[0] for b in BEAM_BAD])
def test_bad_beam_calls_are_refused(L, what, kw, msg):
    a = _args(kw.get("beam", 2))
    if "V" in kw:
        a.V = kw["V"]
    pen = ctypes.byref(_penalty(**kw["pen"])) if "pen" in kw else None
    rc, err = _beam(L, a, ctypes.byref(_layer()), pen, div=kw.get("div", (1.0, 0.0, None, None)))
    assert rc == -1 and msg in err, err


def test_penalty_checks_come_before_the_shared_ones(L):
    """a NULL penalty means none; a good penalty passes on to the shared checks (here: the region offsets)"""
    for pen in (None, ctypes.byref(_penalty())):
        rc, err = _beam(L, _args(2, off=[1, 3, 5, 8]), ctypes.byref(_layer()), pen)
        assert rc == -1 and b"reg_off_host[0] must be 0" in err, err


# ------------------------------------------------------------------------------------------------ the CPU oracle
V = 30
START, END = V - 2, 5


def _setup(seed=3, N=3, R=10):
    from oracle import ref_ext as rx
    from oracle import ref_model as rm
    _, pd = rm.init_params(V, seed=seed, dtype=torch.float64)
    _, p2 = rx.init_params_ext(seed=seed + 1, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = ((torch.rand(V, 512, generator=g) * 2 - 1) * 0.5).double()
    pd["embedding.weight"] = ((torch.rand(V, 512, generator=g) * 2 - 1) * 1.0).double()
    enc = (torch.relu(torch.randn(N, R, 512, generator=g)) * 0.7).double()
    return pd, p2, enc


def test_greedy_logits_are_the_teacher_forced_forward():
    from oracle import ref_ext as rx
    pd, p2, enc = _setup(5)
    ids, logits, att = d2o.greedy_decode(pd, p2, enc, START, END, 9)
    N, n = ids.shape
    assert n >= 2 and logits.shape == (N, n, V) and att.shape == (N, n, enc.shape[1])
    caps = torch.cat([torch.full((N, 1), START, dtype=torch.long), ids[:, :-1]], dim=1)
    preds, alphas = rx.decoder2_forward(pd, p2, enc, caps, n)
    assert (preds - logits).abs().max().item() < 1e-12
    assert (alphas - att).abs().max().item() < 1e-12
    assert torch.equal(preds.argmax(dim=-1), ids)


def test_beam_of_width_one_is_greedy():
    """beam 1 chooses the argmax while a row is unfinished and END after it (greedy keeps decoding): the tokens agree up to
    each row's first END, and both run the same number of steps"""
    pd, p2, enc = _setup(5)
    gids, _, _ = d2o.greedy_decode(pd, p2, enc, START, END, 9)
    for fin in ("reference", "backtrack"):
        bids, _, _ = d2o.beam_decode(pd, p2, enc, START, END, 1, 9, finalize=fin)
        assert bids.shape == (gids.shape[0], gids.shape[1], 1)
        for g, b in zip(gids.tolist(), bids[:, :, 0].tolist()):
            n = g.index(END) + 1 if END in g else len(g)
            assert b[:n] == g[:n] and all(t == END for t in b[n:])
