"""CPU (-m "not gpu"): the length and coverage penalties of beam search (lo_beam_penalty).  The two entry points
lo_decoder_beam_pen / lo_tfdec_beam_pen are bound from the header and refuse every bad penalty with LO_EINVAL before any GPU work;
the penalised CPU search of tests/beam_penalty_oracle.py is the oracles' own search, bit for bit, with both weights 0; and on two
hand-built two-step searches the length penalty, and separately the coverage penalty, changes the chosen hypothesis."""
import ctypes
import math

import pytest
import torch

import beam_penalty_oracle as bpo
from latex_ocr_b200 import _lib, decode, tf_decoder

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000
_TF_BUFFERS = ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init",
               "emb", "formula", "lengths", "loss", "denc", "g_w_img", "g_w_cat2", "g_beta", "g_w_lstm", "g_b_lstm", "g_w_oc", "g_w_y",
               "g_w_init", "g_b_init", "g_emb")


@pytest.fixture
def L():
    return _lib.lib()


def _offsets(a, off):
    if off is not None:
        a._off = (ctypes.c_int32 * len(off))(*off)
        a.reg_off_host = ctypes.cast(a._off, ctypes.c_void_p)
        a.reg_off = _FAKE
    return a


def _args(V, beam, off):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 3 * beam, 3, 8, 512, 512, 512, 512, V
    a.rows_per_img = beam
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = _FAKE
    a._bt = (ctypes.c_int32 * 3)(3, 3, 3)
    a.bt_host = ctypes.cast(a._bt, ctypes.c_void_p)
    return _offsets(a, off)


def _tf_args(V, beam, off):
    a = tf_decoder.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 3 * beam, 3, 8, 512, 256, 512, 512, 80, V
    a.rows_per_img = beam
    a.dt = _lib.LO_F32
    for k in _TF_BUFFERS:
        setattr(a, k, _FAKE)
    a.formula_stride = a.T
    a.inv_n_words = 1.0
    return _offsets(a, off)


def _penalty(**kw):
    p = _lib.BeamPenalty()
    p.alpha, p.beta = 0.6, 0.2
    p.len_pen = p.cov = p.len = p.scores = _FAKE
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _call(L, flavour, pen, V=40, beam=2, off=None):
    o = [ctypes.c_void_p(_FAKE)] * 4
    if flavour == "torch":
        rc = L.lo_decoder_beam_pen(ctypes.byref(_args(V, beam, off)), 0, 1, 3, *o, 1.0, 0.0, None, None, pen, None)
    else:
        rc = L.lo_tfdec_beam_pen(ctypes.byref(_tf_args(V, beam, off)), 1, 3, *o, 1.0, 0.0, None, None, pen, None)
    return rc, L.lo_last_error()


def test_bound_from_the_header(L):
    sigs = _lib.declared_signatures()
    for name, n_args in (("lo_decoder_beam_pen", 14), ("lo_tfdec_beam_pen", 13)):
        restype, argtypes = sigs[name]
        assert restype is ctypes.c_int and len(argtypes) == n_args
        assert argtypes[-2] == ctypes.POINTER(_lib.BeamPenalty)
        assert getattr(L, name).argtypes == argtypes
        # the _div signature plus the penalty
        assert argtypes[:-2] == sigs[name.replace("_pen", "_div")][1][:-1]
    assert L.lo_sizeof_beam_penalty() == ctypes.sizeof(_lib.BeamPenalty)
    assert [f[0] for f in _lib.BeamPenalty._fields_] == ["alpha", "beta", "len_pen", "cov", "len", "scores"]


BAD = [
    ("null struct", None, b"null lo_beam_penalty"),
    ("alpha < 0", dict(alpha=-0.1), b"finite and >= 0"),
    ("beta < 0", dict(beta=-1e-6), b"finite and >= 0"),
    ("alpha nan", dict(alpha=math.nan), b"finite and >= 0"),
    ("alpha inf", dict(alpha=math.inf), b"finite and >= 0"),
    ("beta nan", dict(beta=math.nan), b"finite and >= 0"),
    ("beta inf", dict(beta=math.inf), b"finite and >= 0"),
    ("alpha without len_pen", dict(len_pen=None), b"needs the len_pen table"),
    ("beta without cov", dict(cov=None), b"needs the cov scratch"),
    ("null len", dict(len=None), b"null len scratch"),
    ("null len, no penalty", dict(alpha=0.0, beta=0.0, len=None), b"null len scratch"),
]


@pytest.mark.parametrize("flavour", ["torch", "tf"])
@pytest.mark.parametrize("what,kw,msg", BAD, ids=[b[0] for b in BAD])
def test_bad_penalties_are_refused(L, flavour, what, kw, msg):
    rc, err = _call(L, flavour, None if kw is None else ctypes.byref(_penalty(**kw)))
    assert rc == -1 and msg in err, err


@pytest.mark.parametrize("flavour", ["torch", "tf"])
def test_optional_pointers_may_be_null_when_their_penalty_is_off(L, flavour):
    """alpha = 0 needs no table, beta = 0 no coverage scratch, and scores are optional: such a penalty passes, and the call goes
    on to refuse the (deliberately bad) region offsets"""
    for kw in (dict(alpha=0.0, len_pen=None), dict(beta=0.0, cov=None), dict(scores=None), dict(alpha=0.0, beta=0.0, len_pen=None,
                                                                                                 cov=None, scores=None)):
        rc, err = _call(L, flavour, ctypes.byref(_penalty(**kw)), off=[1, 3, 5, 8])
        assert rc == -1 and b"reg_off_host[0] must be 0" in err, (kw, err)


@pytest.mark.parametrize("flavour", ["torch", "tf"])
def test_the_shared_memory_limit_counts_the_score_array(L, flavour):
    """beam 16 x V 2000: the totals alone fit in 200 kB (what the _div entry points accept), with the scores they do not"""
    rc, err = _call(L, flavour, ctypes.byref(_penalty()), V=2000, beam=16)
    assert rc == -1 and b"beam*V too large" in err
    for kw in (dict(alpha=0.6, beta=0.0), dict(alpha=0.0, beta=0.2)):
        rc, err = _call(L, flavour, ctypes.byref(_penalty(**kw)), V=2000, beam=16)
        assert rc == -1 and b"beam*V too large" in err
    rc, err = _call(L, flavour, ctypes.byref(_penalty(alpha=0.0, beta=0.0)), V=2000, beam=16, off=[1, 3, 5, 8])
    assert rc == -1 and b"reg_off_host[0] must be 0" in err


@pytest.mark.parametrize("flavour", ["torch", "tf"])
def test_beam_above_V_is_refused(L, flavour):
    """time 0 ranks beam 0's V tokens alone: a beam wider than V would repeat a hypothesis, so it is refused, with and without a
    penalty; beam == V passes on to the next check (the deliberately bad region offsets)"""
    for pen in (ctypes.byref(_penalty(alpha=0.0, beta=0.0)), ctypes.byref(_penalty())):
        for beam, V in ((4, 3), (16, 15), (3, 2)):
            rc, err = _call(L, flavour, pen, V=V, beam=beam)
            assert rc == -1 and b"beam (rows_per_img) <= V" in err, (beam, V, err)
        rc, err = _call(L, flavour, pen, V=3, beam=3, off=[1, 3, 5, 8])
        assert rc == -1 and b"reg_off_host[0] must be 0" in err, err
    # the entry points without penalties share the check
    o = [ctypes.c_void_p(_FAKE)] * 4
    if flavour == "torch":
        rc = L.lo_decoder_beam_div(ctypes.byref(_args(3, 4, None)), 0, 1, 3, *o, 1.0, 0.0, None, None, None)
    else:
        rc = L.lo_tfdec_beam_div(ctypes.byref(_tf_args(3, 4, None)), 1, 3, *o, 1.0, 0.0, None, None, None)
    assert rc == -1 and b"beam (rows_per_img) <= V" in L.lo_last_error()


def test_python_refuses_negative_weights():
    for a, b in ((-0.1, 0.0), (0.0, -0.5), (math.nan, 0.0), (0.0, math.inf)):
        with pytest.raises(ValueError):
            decode.penalty_weights(a, b)
    assert decode.penalty_weights(0, 0) == (0.0, 0.0)


def test_length_penalty_table():
    t = decode.length_penalty_table(0.6, 152)
    assert t.dtype == torch.float32 and t.shape == (153,)
    want = [((5.0 + l) / 6.0) ** 0.6 for l in range(153)]
    assert torch.equal(t, torch.tensor(want, dtype=torch.float64).float())
    assert torch.equal(t, bpo.length_penalty_table(0.6, 153))
    assert torch.equal(decode.length_penalty_table(0.0, 10), torch.ones(11))


# ------------------------------------------------------------------------------------------------ the CPU search
V = 30
START, END = V - 2, 5


def _torch_params(seed):
    from oracle import ref_model as rm
    _, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    return pd


def _tf_params(seed):
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(40, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0
    return p


def _enc(N, R, seed):
    return torch.relu(torch.randn(N, R, 512, generator=torch.Generator().manual_seed(seed))) * 0.7


@pytest.mark.parametrize("beam", [1, 3])
@pytest.mark.parametrize("div", [False, True])
def test_zero_penalties_are_the_oracles_search(beam, div):
    from oracle import ref_decode as rd
    from oracle import ref_tf_model as tfm
    max_iter = 7
    N = 3
    pd = _torch_params(3)
    enc = _enc(N, 12, 4)
    kw = dict(div_gamma=0.5, div_prob=0.7, div_u=torch.rand(max_iter + 2, N * beam, V, generator=torch.Generator().manual_seed(5))) \
        if div else {}
    for fin in ("reference", "backtrack"):
        want, wlp = rd.beam_decode(pd, enc, START, END, beam, max_iter, finalize=fin, **kw)
        got, glp, gsc = bpo.beam_decode(pd, enc, START, END, beam, max_iter, finalize=fin, **kw)
        assert torch.equal(got, want) and torch.equal(glp, wlp) and torch.equal(gsc, wlp)
    p = _tf_params(6)
    if div:
        kw["div_u"] = torch.rand(max_iter + 2, N * beam, 40, generator=torch.Generator().manual_seed(7))
    want, wlp = tfm.beam_decode(p, enc, END, beam, max_iter, **kw)
    got, glp, gsc = bpo.tf_beam_decode(p, enc, END, beam, max_iter, **kw)
    assert torch.equal(got, want) and torch.equal(glp, wlp) and torch.equal(gsc, wlp)


def _scripted(step0, step1, alpha0=None, alpha1=None):
    """a cell over V = 3 tokens (0 = END) of one image: log-probs step0 [3] at time 0, then step1[tok] for the token a row was fed;
    attention weights alpha0 [R] at time 0, alpha1[tok] after"""
    def cell(tok):
        if tok is None:
            lp = torch.tensor([step0] * 2)
            a = torch.tensor([alpha0 or [1.0]] * 2)
        else:
            lp = torch.stack([torch.tensor(step1[int(k)]) for k in tok])
            a = torch.stack([torch.tensor((alpha1 or {}).get(int(k), [1.0])) for k in tok])
        return lp.log(), a
    return cell


def test_length_penalty_changes_the_hypothesis():
    """beam 2.  Time 0: END 0.5, a 0.4, b 0.1; after a: END 0.9.  Without the penalty the one-step hypothesis [END] wins; with
    alpha = 3 (LP[0] = (5/6)^3 < 1 inflates it, LP[1] = 1) [a, END] wins, and each keeps its raw log-prob."""
    cell = _scripted([0.5, 0.4, 0.1], {0: [1.0, 1e-9, 1e-9], 1: [0.9, 0.05, 0.05], 2: [0.9, 0.05, 0.05]})
    run = lambda alpha: bpo.search(cell, lambda rows: None, 1, 2, 3, 0, 5, alpha=alpha)
    ids, parents, lp, sc = run(0.0)
    assert ids[0].tolist() == [[0, 1], [0, 0]] and parents[0, 1].tolist() == [0, 1]   # hypothesis 0 = [END]
    ids, parents, lp, sc = run(3.0)
    assert ids[0].tolist() == [[1, 0], [0, 0]] and parents[0, 1].tolist() == [0, 1]   # hypothesis 0 = [a, END]
    l_a_end = math.log(0.4) + math.log(0.9)
    assert abs(lp[0, 0].item() - l_a_end) < 1e-6 and abs(lp[0, 1].item() - math.log(0.5)) < 1e-6
    assert abs(sc[0, 0].item() - l_a_end) < 1e-6                                        # len 1: LP[1] = 1
    assert abs(sc[0, 1].item() - math.log(0.5) / (5 / 6) ** 3) < 1e-5                   # len 0: LP[0]


def test_coverage_penalty_changes_the_hypothesis():
    """beam 2, two regions.  Time 0 attends region 0 (0.9, 0.1): a 0.5, b 0.4.  After a the row attends region 0 again, after b
    region 1; both then end (END 0.9).  Without the penalty [a, END] wins; with beta = 0.5 its coverage (1.8, 0.2) costs
    0.5 ln 0.2 while [b, END] covers both regions (1.0, 1.0) at no cost, and [b, END] wins."""
    cell = _scripted([0.1, 0.5, 0.4], {0: [1.0, 1e-9, 1e-9], 1: [0.9, 0.05, 0.05], 2: [0.9, 0.05, 0.05]},
                     alpha0=[0.9, 0.1], alpha1={0: [0.5, 0.5], 1: [0.9, 0.1], 2: [0.1, 0.9]})
    run = lambda beta: bpo.search(cell, lambda rows: None, 1, 2, 3, 0, 5, beta=beta)
    ids, parents, lp, sc = run(0.0)
    assert ids[0].tolist() == [[1, 2], [0, 0]] and parents[0, 1].tolist() == [0, 1]   # hypothesis 0 = [a, END]
    ids, parents, lp, sc = run(0.5)
    assert ids[0].tolist() == [[1, 2], [0, 0]] and parents[0, 1].tolist() == [1, 0]   # hypothesis 0 = [b, END]
    l_b_end, l_a_end = math.log(0.4) + math.log(0.9), math.log(0.5) + math.log(0.9)
    assert abs(lp[0, 0].item() - l_b_end) < 1e-6 and abs(lp[0, 1].item() - l_a_end) < 1e-6
    assert abs(sc[0, 0].item() - l_b_end) < 1e-5
    assert abs(sc[0, 1].item() - (l_a_end + 0.5 * math.log(0.2))) < 1e-5
