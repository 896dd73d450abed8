"""CPU (-m "not gpu"): decode.BracketRule (the LaTeX builder, check(), the refusals), the lo_bracket_rule binding and the refusals
of the nine *_brackets entry points before any GPU work, and the rule against real formulas: the first 500 lines of the
reference's data/test.formulas.norm.txt (tests/golden/formulas_sample.txt) all pass."""
import ctypes
import os

import pytest
import torch

import bracket_oracle as bo
from latex_ocr_b200 import _lib, decode

HERE = os.path.dirname(os.path.abspath(__file__))
# never dereferenced: every call below is refused before any GPU work
_FAKE = 0x1000

VOCAB = ["_END", "x", "{", "}", "\\leftarrow", "\\rightarrow", "\\left.", "\\right\\}", "\\begin{array}", "\\end{array}",
         "\\begin{foo}", "\\{", "\\}", "(", ")", "[", "]", "\\left(", "\\right)", "\\end{bar}", "\\lefteqn"]
T = {t: i for i, t in enumerate(VOCAB)}


def _ids(s):
    return [T[t] for t in s.split()]


@pytest.fixture
def rule():
    return decode.BracketRule.latex(VOCAB)


def test_latex_roles(rule):
    role = dict(zip(VOCAB, rule.role))
    assert role["{"] == 1 and role["}"] == -1
    assert role["\\left."] == role["\\left("] == 2 and role["\\right\\}"] == role["\\right)"] == -2
    assert role["\\begin{array}"] == 3 and role["\\end{array}"] == -3
    for t in ("_END", "x", "\\leftarrow", "\\rightarrow", "\\lefteqn", "\\begin{foo}", "\\end{bar}", "\\{", "\\}", "(", ")", "[", "]"):
        assert role[t] == 0, t
    assert rule.n_kinds == 3 and rule.max_depth == 16
    # a dict id -> token gives the same table
    assert decode.BracketRule.latex(dict(enumerate(VOCAB))).role == rule.role


def test_check(rule):
    ok = ["x", "{ x } _END x }", "\\left( { x } \\right\\}", "\\left. x \\right)", "\\begin{array} { x } \\end{array}",
          "( ] \\{ \\leftarrow", "", "_END {"]
    bad = ["{", "}", "{ \\right)", "\\left( }", "\\begin{array} { \\end{array} }", "{ x", "\\left( \\begin{array} \\right)"]
    assert rule.check([_ids(s) for s in ok], T["_END"]) == [True] * len(ok)
    assert rule.check([_ids(s) for s in bad], T["_END"]) == [False] * len(bad)
    # tensors of any leading shape
    t = torch.tensor([[_ids("{ x }")[0], T["x"], T["}"]], [T["{"], T["{"], T["}"]]])
    assert rule.check(t, T["_END"]) == [True, False]
    assert rule.check(t.view(1, 2, 3), T["_END"]) == [True, False]
    # deeper than max_depth
    shallow = decode.BracketRule.latex(VOCAB, max_depth=2)
    assert shallow.check([_ids("{ { } }"), _ids("{ { { } } }")], T["_END"]) == [True, False]


def test_refusals():
    with pytest.raises(ValueError, match="out of range"):
        decode.BracketRule([0, 1, -1, 256])
    with pytest.raises(ValueError, match="closing"):
        decode.BracketRule([0, 1, 2, -2])
    with pytest.raises(ValueError, match="opening"):
        decode.BracketRule([0, -1, 2, -2])
    for d in (0, 33):
        with pytest.raises(ValueError, match="max_depth"):
            decode.BracketRule([0, 1, -1], max_depth=d)
    r = decode.BracketRule([0, 1, -1, 0])
    with pytest.raises(ValueError, match="END"):
        r.args(1, 4, 2, 10, "cpu")
    with pytest.raises(ValueError, match="entries"):
        r.args(0, 5, 2, 10, "cpu")
    # step 0 allows END, the neutral token and the open: 3 tokens, so beam 4 is refused
    assert r.allowed_at_start(0, 10) == 3 and r.allowed_at_start(0, 1) == 2
    with pytest.raises(ValueError, match="beam_size"):
        r.args(0, 4, 8, 10, "cpu", beam=4)
    with pytest.raises(ValueError, match="backtrack"):
        decode.refuse_reference_finalize(r, "reference")
    decode.refuse_reference_finalize(None, "reference")
    with pytest.raises(TypeError):
        decode.bracket_args([0, 1, -1], 0, 3, 2, 10, "cpu")
    assert decode.bracket_args(None, 0, 3, 2, 10, "cpu") == (None, None)
    decode.BracketRule([0] * 5)              # no kinds: accepted


def test_real_formulas_pass():
    lines = [l for l in open(os.path.join(HERE, "golden", "formulas_sample.txt"), encoding="utf-8").read().split("\n") if l.strip()]
    assert len(lines) == 500
    toks = sorted({t for l in lines for t in l.split()})
    vocab = ["_END"] + toks
    ids = {t: i for i, t in enumerate(vocab)}
    rule = decode.BracketRule.latex(vocab)
    assert rule.n_kinds >= 3
    seqs = [[ids[t] for t in l.split()] for l in lines]
    assert all(rule.check(seqs, 0))
    # and the rule bites on them: dropping the last closing token of a formula that has one breaks it
    cut = [s[:max(i for i, v in enumerate(s) if rule.role[v] < 0)] for s in seqs if any(rule.role[v] < 0 for v in s)]
    assert cut and not any(rule.check(cut, 0))


def test_oracle_greedy_under_the_rule_is_well_formed(rule):
    """tests/bracket_oracle.py on a cell that always prefers an opening token: every row closes before its last step"""
    V, B = len(VOCAB), 4
    g = torch.Generator().manual_seed(0)

    def cell(tok):
        x = torch.randn(B, V, generator=g, dtype=torch.float64)
        x[:, T["{"]] += 5.0
        x[:, T["\\left("]] += 4.0
        return x
    for L in (1, 2, 5, 9):
        ids = bo.greedy(cell, B, rule, T["_END"], L)
        assert all(rule.check(ids, T["_END"]))
        assert (ids == T["{"]).any() or L < 2


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture
def L():
    return _lib.lib()


def test_mirror_matches_the_library(L):
    assert L.lo_sizeof_bracket_rule() == ctypes.sizeof(_lib.BracketRule)
    assert [f[0] for f in _lib.BracketRule._fields_] == ["role", "n_kinds", "max_depth", "state"]
    assert L.lo_bracket_state_bytes(10, 16) >= 10 * 8 + 2 * 10 * 16
    assert L.lo_bracket_state_bytes(0, 16) == 0 and L.lo_bracket_state_bytes(4, 33) == 0


def _dec_args():
    a = _lib.DecoderArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.E, a.V = 2, 3, 8, 512, 512, 512, 512, 40
    a.dt = _lib.LO_F32
    a.caps = a.enc = a.work = a.dlogits = _FAKE
    a.rows_per_img = 1
    bt = (ctypes.c_int32 * 3)(2, 2, 2)
    a.bt_host = ctypes.cast(bt, ctypes.c_void_p)
    return a, bt


def _tf_args():
    from latex_ocr_b200 import tf_decoder
    a = tf_decoder.TfDecArgs()
    a.V, a.rows_per_img = 40, 1
    return a


def _sample():
    s = _lib.SampleArgs()
    s.tau, s.top_k, s.top_p, s.u, s.logp = 1.0, 0, 1.0, _FAKE, _FAKE
    return s


def _layer2():
    l2 = _lib.Decoder2Layer()
    l2.w_ih = l2.w_hh = l2.b_ih = l2.b_hh = l2.scratch = _FAKE
    return l2


def _calls(L, br):
    """the nine entry points with fake args (the TF ones with only V and rows_per_img set: the rule is checked before the rest)"""
    a, bt = _dec_args()
    t = _tf_args()
    s, l2 = _sample(), _layer2()
    F = ctypes.c_void_p(_FAKE)
    b = ctypes.byref(br) if br is not None else None
    return [
        lambda: L.lo_decoder_greedy_brackets(ctypes.byref(a), 0, 1, 3, F, F, None, b, None),
        lambda: L.lo_decoder_sample_brackets(ctypes.byref(a), ctypes.byref(s), 0, 1, 3, F, F, None, b, None),
        lambda: L.lo_decoder_beam_brackets(ctypes.byref(a), 0, 1, 3, F, F, F, F, 1.0, 0.0, None, None, None, b, None),
        lambda: L.lo_tfdec_greedy_brackets(ctypes.byref(t), 1, 3, F, None, b, None),
        lambda: L.lo_tfdec_sample_brackets(ctypes.byref(t), ctypes.byref(s), 1, 3, F, None, b, None),
        lambda: L.lo_tfdec_beam_brackets(ctypes.byref(t), 1, 3, F, F, F, F, 1.0, 0.0, None, None, None, b, None),
        lambda: L.lo_decoder2_greedy_brackets(ctypes.byref(a), ctypes.byref(l2), 0, 1, 3, F, F, None, b, None),
        lambda: L.lo_decoder2_sample_brackets(ctypes.byref(a), ctypes.byref(l2), ctypes.byref(s), 0, 1, 3, F, F, None, b, None),
        lambda: L.lo_decoder2_beam_brackets(ctypes.byref(a), ctypes.byref(l2), 0, 1, 3, F, F, F, F, 1.0, 0.0, None, None, None, b,
                                            None),
    ], (a, bt, t, s, l2)


def _rule_struct(**kw):
    br = _lib.BracketRule()
    br.role, br.n_kinds, br.max_depth, br.state = _FAKE, 3, 16, _FAKE
    for k, v in kw.items():
        setattr(br, k, v)
    return br


@pytest.mark.parametrize("bad,msg", [(None, b"null lo_bracket_rule"), (dict(role=None), b"null role"),
                                     (dict(state=None), b"null role table or state"), (dict(n_kinds=0), b"n_kinds"),
                                     (dict(n_kinds=256), b"n_kinds"), (dict(max_depth=0), b"max_depth"),
                                     (dict(max_depth=33), b"max_depth")])
def test_entry_points_refuse_a_bad_rule(L, bad, msg):
    br = None if bad is None else _rule_struct(**bad)
    calls, keep = _calls(L, br)
    for i, call in enumerate(calls):
        rc = call()
        assert rc == -1 and msg in L.lo_last_error(), (i, L.lo_last_error())


def test_entry_points_refuse_a_large_vocabulary(L):
    calls, (a, bt, t, s, l2) = _calls(L, _rule_struct())
    a.V = t.V = 24577
    for i in (0, 2, 3, 5, 6, 8):                    # the sampling entry points refuse V above 2048 first
        rc = calls[i]()
        assert rc == -1 and b"24576" in L.lo_last_error(), (i, L.lo_last_error())
