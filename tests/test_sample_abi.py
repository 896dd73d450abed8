"""CPU (-m "not gpu"): sampling decode (lo_sample_args; lo_decoder_sample, lo_tfdec_sample, lo_decoder2_sample).  The struct and
the three entry points are bound from the header; every bad call is refused with LO_EINVAL before anything is enqueued; the
filter rule of tests/sample_oracle.py (which the GPU tests hold the kernel to) on hand-built rows; and decode.mbr_select's rule on
hand-built similarities."""
import ctypes
import math

import numpy as np
import pytest
import torch

import sample_oracle as so
from latex_ocr_b200 import _lib, decode

# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000
V = 40


@pytest.fixture
def L():
    return _lib.lib()


def _targs(rpi, **kw):
    a = _lib.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = 3 * rpi, 3, 8, 512, 512, 512, 512, 80, V
    a.rows_per_img = rpi
    a.dt = _lib.LO_F32
    for k in ("enc", "ws", "logits", "alphas", "w_img", "w_cat2", "beta", "w_lstm", "b_lstm", "w_oc", "w_y", "w_init", "b_init",
              "emb"):
        setattr(a, k, _FAKE)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _dargs(rpi, **kw):
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 3 * max(rpi, 1), 3, 8, 512, 512, 512, 512, V
    a.rows_per_img = rpi
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = a.row_loss = _FAKE
    a._bt = (ctypes.c_int32 * 3)(a.B, a.B, a.B)
    a.bt_host = ctypes.cast(a._bt, ctypes.c_void_p)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _sample(**kw):
    s = _lib.SampleArgs()
    s.tau, s.top_k, s.top_p = 1.0, 0, 1.0
    s.state = s.logp = _FAKE
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _call(L, entry, a, s, max_steps=3):
    o = [ctypes.c_void_p(_FAKE)] * 3
    a = ctypes.byref(a) if a is not None else None
    s = ctypes.byref(s) if s is not None else None
    if entry == "torch":
        return L.lo_decoder_sample(a, s, 0, 1, max_steps, *o, None)
    if entry == "tf":
        return L.lo_tfdec_sample(a, s, 1, max_steps, o[0], o[1], None)
    l2 = _lib.Decoder2Layer()
    l2.w_ih = l2.w_hh = l2.b_ih = l2.b_hh = l2.scratch = _FAKE
    return L.lo_decoder2_sample(a, ctypes.byref(l2), s, 0, 1, max_steps, *o, None)


def test_bound_from_the_header(L):
    assert [f[0] for f in _lib.SampleArgs._fields_] == ["tau", "top_k", "top_p", "u", "state", "logp"]
    assert L.lo_sizeof_sample_args() == ctypes.sizeof(_lib.SampleArgs)
    sigs = _lib.declared_signatures()
    sp = ctypes.POINTER(_lib.SampleArgs)
    for name, base, at in (("lo_decoder_sample", "lo_decoder_greedy_hist", 1), ("lo_tfdec_sample", "lo_tfdec_greedy", 1),
                           ("lo_decoder2_sample", "lo_decoder2_greedy", 2)):
        restype, argtypes = sigs[name]
        want = list(sigs[base][1])
        assert restype is ctypes.c_int and argtypes == want[:at] + [sp] + want[at:], name
        assert getattr(L, name).argtypes == argtypes


# (name, lo_sample_args fields, args fields, expected message)
BAD = [
    ("null struct", None, {}, b"null lo_sample_args"),
    ("tau 0", dict(tau=0.0), {}, b"temperature"),
    ("tau negative", dict(tau=-1.0), {}, b"temperature"),
    ("tau inf", dict(tau=math.inf), {}, b"temperature"),
    ("tau nan", dict(tau=math.nan), {}, b"temperature"),
    ("top_k negative", dict(top_k=-1), {}, b"top_k"),
    ("top_k above V", dict(top_k=V + 1), {}, b"top_k"),
    ("top_p 0", dict(top_p=0.0), {}, b"top_p"),
    ("top_p above 1", dict(top_p=1.5), {}, b"top_p"),
    ("top_p nan", dict(top_p=math.nan), {}, b"top_p"),
    ("neither u nor state", dict(state=None), {}, b"needs injected uniforms u or the Philox state"),
    ("null logp", dict(logp=None), {}, b"null logp"),
    ("rows_per_img 0", {}, dict(rows_per_img=0), b"rows_per_img"),
    ("rows_per_img 17", {}, dict(rows_per_img=17), b"rows_per_img"),
    ("V above 2048", dict(top_k=0), dict(V=2049), b"V above 2048"),
    ("ss_prob", {}, dict(ss_prob=_FAKE, fed=_FAKE, ss_u=_FAKE), b"scheduled sampling"),
    ("ss_u", {}, dict(ss_u=_FAKE), b"scheduled sampling"),
    ("ss_temp", {}, dict(ss_temp=_FAKE), b"ss_temp"),
    ("ss_gu", {}, dict(ss_gu=_FAKE), b"ss_"),
    ("max_steps above T", {}, dict(max_steps=4), b"max_steps"),
    ("null enc", {}, dict(enc=None), b"null"),
    ("null args", {}, dict(args=None), b"null args"),
]


@pytest.mark.parametrize("entry", ["torch", "tf", "decoder2"])
@pytest.mark.parametrize("what,skw,akw,msg", BAD, ids=[b[0] for b in BAD])
def test_bad_calls_are_refused(L, entry, what, skw, akw, msg):
    akw = dict(akw)
    max_steps = akw.pop("max_steps", 3)
    has_args = akw.pop("args", True)
    rpi = akw.pop("rows_per_img", 2)
    if entry == "tf":
        akw = {k: v for k, v in akw.items() if k not in ("fed",)}
        a = _targs(max(rpi, 1), **akw)
        a.rows_per_img = rpi
    else:
        a = _dargs(rpi, **akw)
    s = _sample(**skw) if skw is not None else None
    before = L.lo_launch_count()
    rc = _call(L, entry, a if has_args else None, s, max_steps)
    assert rc == -1, (entry, what)
    assert msg in L.lo_last_error(), (entry, what, L.lo_last_error())
    assert L.lo_launch_count() == before


# ------------------------------------------------------------------------------------------------ the oracle's filter rule
def test_ties_in_q_keep_the_lower_index_first():
    x = np.array([1.0, 3.0, 2.0, 3.0, 0.5])
    kept, _ = so.keep_mask(x, 1.0, 1, 1.0)
    assert kept.tolist() == [False, True, False, False, False]
    kept, _ = so.keep_mask(x, 0.7, 2, 1.0)
    assert kept.tolist() == [False, True, False, True, False]
    kept, _ = so.keep_mask(x, 1.0, 3, 1.0)
    assert kept.tolist() == [False, True, True, True, False]


def test_top_k_1_is_the_argmax_whatever_the_uniforms():
    g = np.random.default_rng(3)
    for _ in range(20):
        x = g.normal(size=30)
        kept, _ = so.keep_mask(x, 1.3, 1, 1.0)
        assert so.draw(x, 1.3, kept, g.uniform(1e-6, 1 - 1e-6, size=30)) == int(np.argmax(x))


def test_top_p_boundary():
    """q = (0.5, 0.3, 0.15, 0.05): the masses before the tokens are 0, 0.5, 0.8, 0.95"""
    x = np.log(np.array([0.15, 0.5, 0.05, 0.3]))
    for p, want in ((0.4, [1]), (0.499, [1]), (0.501, [1, 3]), (0.799, [1, 3]), (0.801, [1, 3, 0]), (0.951, [1, 3, 0, 2]),
                    (1.0, [0, 1, 2, 3])):
        kept, margin = so.keep_mask(x, 1.0, 0, p)
        assert sorted(np.nonzero(kept)[0].tolist()) == sorted(want), p
        assert margin == (math.inf if p == 1.0 else pytest.approx(min(abs(m - p) for m in (0, 0.5, 0.8, 0.95))))
    # a temperature changes the masses: tau = 2 flattens q to (0.379, 0.294, 0.208, 0.120), masses before 0, 0.379, 0.673, 0.880
    assert sorted(np.nonzero(so.keep_mask(x, 2.0, 0, 0.65)[0])[0].tolist()) == [1, 3]
    assert sorted(np.nonzero(so.keep_mask(x, 2.0, 0, 0.7)[0])[0].tolist()) == [0, 1, 3]


def test_both_filters_together():
    x = np.log(np.array([0.15, 0.5, 0.05, 0.3]))
    assert np.nonzero(so.keep_mask(x, 1.0, 2, 0.9)[0])[0].tolist() == [1, 3]          # top-k binds
    assert np.nonzero(so.keep_mask(x, 1.0, 3, 0.6)[0])[0].tolist() == [1, 3]          # top-p binds
    assert np.nonzero(so.keep_mask(x, 1.0, 1, 0.9)[0])[0].tolist() == [1]


def test_draw_is_the_gumbel_argmax_over_the_kept_set():
    x = np.array([0.0, 1.0, 2.0])
    u = np.array([0.999999, 0.5, 0.01])     # token 0 has the largest noise, token 2 the smallest
    assert so.draw(x, 1.0, np.ones(3, bool), u) == 0
    assert so.draw(x, 1.0, np.array([False, True, True]), u) == 1
    # equal scores: the lower index
    assert so.draw(np.array([1.0, 1.0]), 1.0, np.ones(2, bool), np.array([0.3, 0.3])) == 0


def test_search_finishes_rows_at_end_and_stops_adding():
    """a cell whose row 0 always prefers END (token 1) and row 1 never: row 0 emits END, then END, and its log-prob is one step's"""
    x = torch.tensor([[0.0, 5.0, 0.0], [5.0, -5.0, 0.0]])
    ids, lp, _ = so.search(lambda tok: x, 2, 1, 3, 1.0, 1, 1.0, torch.full((5, 2, 3), 0.5))
    assert ids.tolist() == [[1, 1, 1, 1], [0, 0, 0, 0]]
    ls = torch.log_softmax(x.double(), -1)
    assert lp[0].item() == pytest.approx(ls[0, 1].item()) and lp[1].item() == pytest.approx(4 * ls[1, 0].item())


# ------------------------------------------------------------------------------------------------ mbr_select's rule
def _mbr_rule(ids, end_id):
    """the rule restated with a CPU Levenshtein"""
    def trunc(s):
        s = [int(t) for t in s]
        return s[:s.index(end_id)] if end_id in s else s

    def lev(a, b):
        d = list(range(len(b) + 1))
        for i, x in enumerate(a, 1):
            prev, d[0] = d[0], i
            for j, y in enumerate(b, 1):
                prev, d[j] = d[j], min(d[j] + 1, d[j - 1] + 1, prev + (x != y))
        return d[len(b)]

    def r(a, b):
        a, b = trunc(a), trunc(b)
        return 1.0 if not a and not b else 1.0 - lev(a, b) / max(len(a), len(b))
    N, n, _ = ids.shape
    means = [[sum(r(ids[i, k], ids[i, j]) for j in range(n) if j != k) / (n - 1) for k in range(n)] for i in range(N)]
    return means


def test_mbr_rule_on_hand_built_hypotheses():
    END = 9
    ids = torch.tensor([[[1, 2, 3, END], [1, 2, 4, END], [1, 2, 3, END], [7, 7, END, END]],      # two equal best: index 0
                        [[5, END, 0, 0], [5, 6, END, 0], [5, 6, END, 0], [5, 6, 7, END]]])    # 1 and 2 tie: index 1
    means = _mbr_rule(ids, END)
    assert means[0][0] == means[0][2] > max(means[0][1], means[0][3])
    assert means[1][1] == means[1][2] > max(means[1][0], means[1][3])
    for i, want in ((0, 0), (1, 1)):
        m = means[i]
        assert m.index(max(m)) == want


def test_mbr_one_sample_is_choice_0_agreement_1():
    choice, agree = decode.mbr_select(torch.tensor([[[3, 4, 1]], [[2, 1, 1]]]), 1)
    assert choice.tolist() == [0, 0] and agree.tolist() == [1.0, 1.0]
    assert choice.dtype == torch.int64 and agree.dtype == torch.float32
