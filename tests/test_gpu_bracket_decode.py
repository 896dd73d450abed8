"""-m gpu: balanced brackets in greedy, beam and sampling decode (the *_brackets entry points, decode.BracketRule) in all three
decoder flavours, against the CPU oracles under the same rule (tests/bracket_oracle.py).

The models are random-init with the fc bias of ``{`` and of ``\\left(`` raised, so that the decode without the rule opens brackets it
never closes: every case first checks that the unconstrained output fails BracketRule.check, so the rule has something to do.
fp32: ids equal the float64 oracle's, log-probs within the tolerances of the flavours' existing decode tests (beam 1e-3 relative,
sampling 1e-5); bf16: every output passes check().  The vocabulary is synthetic: tokens named t<i>, with the bracket tokens
below."""
import numpy as np
import pytest
import torch

import bracket_oracle as bo
from util import Cfg, build_model

pytestmark = pytest.mark.gpu

V, TF_V = 30, 40
START, END = V - 2, 5
LEN = 8
OPEN, CLOSE, LEFT, RIGHT, RIGHT_DOT, BEGIN, ENDENV = 10, 11, 12, 13, 14, 15, 16
SPECIAL = {OPEN: "{", CLOSE: "}", LEFT: "\\left(", RIGHT: "\\right)", RIGHT_DOT: "\\right.", BEGIN: "\\begin{array}",
           ENDENV: "\\end{array}", 17: "\\leftarrow", 18: "\\{"}


def _toks(n):
    return [SPECIAL.get(i, "t%d" % i) for i in range(n)]


def _rule(n=V, max_depth=16):
    from latex_ocr_b200 import decode
    return decode.BracketRule.latex(_toks(n), max_depth)


def _rel(got, want):
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).double()
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())


def _d(p):
    return {k: v.double() for k, v in p.items()}


def _u(steps, B, Vv, seed):
    return torch.rand(steps, B, Vv, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).clamp_(1e-6, 1 - 1e-6).float()


def _bites(rule, ids):
    """the unconstrained output is ill-formed somewhere"""
    assert not all(rule.check(ids, END))


def _ok(rule, ids):
    assert all(rule.check(ids, END))


# ------------------------------------------------------------------------------------------------ models
def _torch_params(seed, Vv=V, bias=(3.0, 2.0)):
    from oracle import ref_model as rm
    pe, pd = rm.init_params(Vv, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(Vv, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(Vv, 512, generator=g) * 2 - 1) * 1.0
    pd["fc.bias"][OPEN] += bias[0]
    pd["fc.bias"][LEFT] += bias[1]
    return pe, pd


def _ext_params(seed, bias=(3.0, 2.0)):
    from oracle import ref_ext as rx
    pe, pd = _torch_params(seed, V, bias)
    prow, p2 = rx.init_params_ext(seed=seed + 1)
    return pe, prow, pd, p2


def _ext_model(params, precision):
    from latex_ocr_b200.ext import Img2SeqRowModel
    pe, prow, pd, p2 = params
    m = Img2SeqRowModel(Cfg(), n_tok=V, device="cuda", precision=precision, impl="tc" if precision == "bf16" else "simt")
    m.build_train()
    m.encoder.load_state_dict(pe)
    m.decoder.load_state_dict(pd)
    m.row_encoder.load_state_dict(prow)
    m.layer2.load_state_dict(p2)
    m.train_mode(False)
    return m


def _tf_params(seed):
    """the Genthial head has no bias: ``{`` and ``\\left(`` get scaled copies of the column of the token the model's greedy decode
    emits most, so that they win where it would"""
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(TF_V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0
    top = int(torch.mode(tfm.greedy_decode(p, _tf_enc(6, 12, 8), END, LEN + 1).flatten()).values)
    p["y_W_o"][:, OPEN] = p["y_W_o"][:, top] * 1.1
    p["y_W_o"][:, LEFT] = p["y_W_o"][:, top] * 1.05
    return p


def _tf_decoder(p, decoding="greedy", beam=3, precision="fp32", max_len=LEN, **kw):
    from latex_ocr_b200.tf_decoder import Decoder
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=max_len,
              decoding=decoding, beam_size=beam, **kw)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision=precision, impl="simt" if precision == "fp32" else "tc")
    dec.load_tf_variables(p)
    return dec


def _tf_enc(N, R, seed):
    return torch.relu(torch.randn(N, R, 512, generator=torch.Generator().manual_seed(seed))) * 0.7


@pytest.fixture(scope="module")
def torch_setup():
    from oracle import ref_model as rm
    pe, pd = _torch_params(21)
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=3)
    enc = rm.encoder_forward(_d(pe), img.double()).reshape(img.shape[0], -1, 512)
    return pe, pd, img, enc, build_model(V, pe, pd, "fp32")


@pytest.fixture(scope="module")
def ext_setup():
    import decoder2_decode_oracle as d2o
    from oracle import ref_model as rm
    params = _ext_params(21)
    pe, prow, pd, p2 = params
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=3)
    return params, img, d2o.encode(_d(pe), _d(prow), img.double()), _ext_model(params, "fp32")


def _tf_p():
    if "tf" not in _tf_p.__dict__:
        _tf_p.tf = _tf_params(7)
    return _tf_p.tf


# ------------------------------------------------------------------------------------------------ fp32 against the oracle
BEAM_CASES = [dict(), dict(length_penalty=0.6, coverage_penalty=0.4), dict(div=True), dict(div=True, length_penalty=0.6)]


def _beam_kw(case, B, Vv):
    kw = {k: v for k, v in case.items() if k != "div"}
    okw = dict(alpha=kw.get("length_penalty", 0.0), beta=kw.get("coverage_penalty", 0.0))
    if case.get("div"):
        u = torch.rand(LEN + 2, B, Vv, generator=torch.Generator().manual_seed(77))
        kw.update(div_gamma=0.5, div_prob=0.7, div_u=u)
        okw.update(div_gamma=0.5, div_prob=0.7, div_u=u.double())
    return kw, okw


def test_torch_greedy(torch_setup):
    from latex_ocr_b200 import decode
    pe, pd, img, enc, m = torch_setup
    rule = _rule()
    _bites(rule, decode.greedy_decode(m, img, START, END, LEN))
    cell, _ = bo.torch_cells(_d(pd), enc, 1, START)
    want = bo.greedy(bo.first(cell), img.shape[0], rule, END, LEN + 1)
    ids = decode.greedy_decode(m, img, START, END, LEN, brackets=rule)
    assert torch.equal(ids, want)
    _ok(rule, ids)


@pytest.mark.parametrize("case", range(len(BEAM_CASES)))
def test_torch_beam(torch_setup, case):
    from latex_ocr_b200 import decode
    pe, pd, img, enc, m = torch_setup
    rule, beam = _rule(), 3
    kw, okw = _beam_kw(BEAM_CASES[case], img.shape[0] * beam, V)
    free, _ = decode.beam_decode(m, img, START, END, beam, LEN, finalize="backtrack", **kw)
    _bites(rule, free)
    cell, reorder = bo.torch_cells(_d(pd), enc, beam, START)
    want, wlp, _ = bo.beam(cell, reorder, img.shape[0], beam, V, rule, END, LEN + 1, **okw)
    ids, lp = decode.beam_decode(m, img, START, END, beam, LEN, finalize="backtrack", brackets=rule, **kw)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3 and torch.isfinite(lp).all()
    _ok(rule, ids)


@pytest.mark.parametrize("tau,k,p", [(1.0, 0, 1.0), (0.7, 5, 1.0), (1.3, 0, 0.7)])
def test_torch_sample(torch_setup, tau, k, p):
    from latex_ocr_b200 import decode
    pe, pd, img, enc, m = torch_setup
    rule, n = _rule(), 4
    u = _u(LEN + 2, img.shape[0] * n, V, 11)
    free, _ = decode.sample_decode(m, img, START, END, n, tau, k, p, LEN, u=u)
    _bites(rule, free)
    cell, _ = bo.torch_cells(_d(pd), enc, n, START)
    want, wlp, margin = bo.sample(bo.first(cell), img.shape[0] * n, rule, END, LEN + 1, tau, k, p, u)
    assert margin >= 1e-4
    ids, lp = decode.sample_decode(m, img, START, END, n, tau, k, p, LEN, u=u, brackets=rule)
    assert torch.equal(ids.reshape(-1, ids.shape[2]), want)
    assert _rel(lp.reshape(-1), wlp) < 1e-5 and torch.isfinite(lp).all()
    _ok(rule, ids)


def test_tf_greedy():
    p, rule = _tf_p(), _rule(TF_V)
    enc = _tf_enc(6, 12, 8)
    dec = _tf_decoder(p)
    _bites(rule, dec.decode(enc.cuda()).ids.cpu())
    cell, _ = bo.tf_cells(_d(p), enc.double(), 1)
    want = bo.greedy(bo.first(cell), 6, rule, END, LEN + 1)
    ids = dec.decode(enc.cuda(), brackets=rule).ids.cpu()
    assert torch.equal(ids, want)
    _ok(rule, ids)


@pytest.mark.parametrize("case", range(len(BEAM_CASES)))
def test_tf_beam(case):
    p, rule, beam = _tf_p(), _rule(TF_V), 3
    enc = _tf_enc(6, 12, 8)
    kw, okw = _beam_kw(BEAM_CASES[case], 6 * beam, TF_V)
    div_u = kw.pop("div_u", None)
    dec = _tf_decoder(p, "beam_search", beam, **kw)
    free = dec.decode(enc.cuda(), div_u=div_u, finalize="backtrack").ids.cpu()
    _bites(rule, free.permute(0, 2, 1))
    cell, reorder = bo.tf_cells(_d(p), enc.double(), beam)
    want, wlp, _ = bo.beam(cell, reorder, 6, beam, TF_V, rule, END, LEN + 1, **okw)
    out, lp = dec.decode(enc.cuda(), div_u=div_u, finalize="backtrack", return_log_probs=True, brackets=rule)
    assert torch.equal(out.ids.cpu(), want)
    assert _rel(lp, wlp) < 1e-3 and torch.isfinite(lp).all()
    _ok(rule, out.ids.cpu().permute(0, 2, 1))


@pytest.mark.parametrize("tau,k,p", [(1.0, 0, 1.0), (0.7, 5, 1.0)])
def test_tf_sample(tau, k, p):
    tp, rule, n = _tf_p(), _rule(TF_V), 4
    enc = _tf_enc(6, 12, 8)
    u = _u(LEN + 2, 6 * n, TF_V, 12)
    dec = _tf_decoder(tp)
    _bites(rule, dec.sample(enc.cuda(), n, tau, k, p, u=u)[0].cpu())
    cell, _ = bo.tf_cells(_d(tp), enc.double(), n)
    want, wlp, _ = bo.sample(bo.first(cell), 6 * n, rule, END, LEN + 1, tau, k, p, u)
    ids, lp = dec.sample(enc.cuda(), n, tau, k, p, u=u, brackets=rule)
    assert torch.equal(ids.cpu().reshape(-1, ids.shape[2]), want)
    assert _rel(lp.reshape(-1), wlp) < 1e-5
    _ok(rule, ids.cpu())


def test_ext_greedy(ext_setup):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), img, enc, m = ext_setup
    rule = _rule()
    _bites(rule, ext.greedy_decode(m, img, START, END, LEN))
    cell, _ = bo.decoder2_cells(_d(pd), _d(p2), enc, 1, START)
    want = bo.greedy(bo.first(cell), img.shape[0], rule, END, LEN + 1)
    ids = ext.greedy_decode(m, img, START, END, LEN, brackets=rule)
    assert torch.equal(ids, want)
    _ok(rule, ids)


@pytest.mark.parametrize("case", range(len(BEAM_CASES)))
def test_ext_beam(ext_setup, case):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), img, enc, m = ext_setup
    rule, beam = _rule(), 3
    kw, okw = _beam_kw(BEAM_CASES[case], img.shape[0] * beam, V)
    free, _ = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, finalize="backtrack", **kw)
    _bites(rule, free)
    cell, reorder = bo.decoder2_cells(_d(pd), _d(p2), enc, beam, START)
    want, wlp, _ = bo.beam(cell, reorder, img.shape[0], beam, V, rule, END, LEN + 1, **okw)
    ids, lp = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, finalize="backtrack", brackets=rule, **kw)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3
    _ok(rule, ids)


@pytest.mark.parametrize("tau,k,p", [(1.0, 0, 1.0), (0.7, 5, 1.0)])
def test_ext_sample(ext_setup, tau, k, p):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), img, enc, m = ext_setup
    rule, n = _rule(), 4
    u = _u(LEN + 2, img.shape[0] * n, V, 13)
    _bites(rule, ext.sample_decode(m, img, START, END, n, temperature=tau, top_k=k, top_p=p, max_length_formula=LEN, u=u)[0])
    cell, _ = bo.decoder2_cells(_d(pd), _d(p2), enc, n, START)
    want, wlp, _ = bo.sample(bo.first(cell), img.shape[0] * n, rule, END, LEN + 1, tau, k, p, u)
    ids, lp = ext.sample_decode(m, img, START, END, n, temperature=tau, top_k=k, top_p=p, max_length_formula=LEN, u=u,
                                brackets=rule)
    assert torch.equal(ids.reshape(-1, ids.shape[2]), want)
    assert _rel(lp.reshape(-1), wlp) < 1e-5
    _ok(rule, ids)


# ------------------------------------------------------------------------------------------------ invariants
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_every_output_is_well_formed(torch_setup, ext_setup, precision):
    """greedy, beam (backtrack, with penalties) and sampling (Philox) of all three flavours, fp32 and bf16: every output passes"""
    from latex_ocr_b200 import decode, ext
    pe, pd, img, _, _ = torch_setup
    m = build_model(V, pe, pd, precision, impl="tc" if precision == "bf16" else "simt")
    em = _ext_model(ext_setup[0], precision)
    rule = _rule()
    for mod, model in ((decode, m), (ext, em)):
        _ok(rule, mod.greedy_decode(model, img, START, END, LEN, brackets=rule))
        ids, lp = mod.beam_decode(model, img, START, END, 5, max_length_formula=LEN, finalize="backtrack", brackets=rule,
                                  length_penalty=0.6, coverage_penalty=0.4)
        _ok(rule, ids)
        assert torch.isfinite(lp).all()
        ids, lp = mod.sample_decode(model, img, START, END, 8, top_p=0.9, max_length_formula=LEN, seed=5, brackets=rule)
        _ok(rule, ids)
        assert torch.isfinite(lp).all()
    tr = _rule(TF_V)
    enc = _tf_enc(6, 12, 8).cuda()
    _ok(tr, _tf_decoder(_tf_p(), precision=precision).decode(enc, brackets=tr).ids.cpu())
    out, lp = _tf_decoder(_tf_p(), "beam_search", 5, precision=precision).decode(enc, finalize="backtrack", return_log_probs=True,
                                                                                  brackets=tr)
    _ok(tr, out.ids.cpu().permute(0, 2, 1))
    assert torch.isfinite(lp).all()
    ids, lp = _tf_decoder(_tf_p(), precision=precision).sample(enc, 8, seed=3, brackets=tr)
    _ok(tr, ids.cpu())
    assert torch.isfinite(lp).all()


@pytest.mark.parametrize("L", [4, 5, 6])
def test_small_cap_closes_everything(L):
    """a model biased hard to open, max_length_formula 4..6: the rule still closes every bracket before the last step"""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    pe, pd = _torch_params(5, bias=(6.0, 5.0))
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=4)
    m = build_model(V, pe, pd, "fp32")
    rule = _rule(max_depth=3)
    _bites(rule, decode.greedy_decode(m, img, START, END, L))
    g = decode.greedy_decode(m, img, START, END, L, brackets=rule)
    _ok(rule, g)
    assert (g == OPEN).any() or (g == LEFT).any()
    _ok(rule, decode.beam_decode(m, img, START, END, 4, L, finalize="backtrack", brackets=rule)[0])
    _ok(rule, decode.sample_decode(m, img, START, END, 8, max_length_formula=L, seed=2, brackets=rule)[0])
    tr = _rule(TF_V, max_depth=3)
    _ok(tr, _tf_decoder(_tf_p(), max_len=L).decode(_tf_enc(6, 12, 8).cuda(), brackets=tr).ids.cpu())


def test_ragged_list(torch_setup):
    """images of different sizes in one call: each image's output is the one it gets decoded alone, and well-formed"""
    from latex_ocr_b200 import _lib, decode
    from oracle import ref_model as rm
    pe, pd, _, _, m = torch_setup
    rule = _rule()
    shapes = ((32, 64), (48, 96), (32, 200))
    imgs = [rm.synthetic_batch(1, H, W, V, 3, 5, seed=40 + k)[0][0] for k, (H, W) in enumerate(shapes) for _ in range(2)]
    with _lib.option(att_nsplit=3):
        g = decode.greedy_decode(m, imgs, START, END, LEN, brackets=rule)
        b, blp = decode.beam_decode(m, imgs, START, END, 3, LEN, finalize="backtrack", brackets=rule)
        s, slp = decode.sample_decode(m, imgs, START, END, 4, max_length_formula=LEN, seed=9, brackets=rule)
        for x in (g, b, s):
            _ok(rule, x)
        for i in (0, 3, 5):
            g1 = decode.greedy_decode(m, [imgs[i]], START, END, LEN, brackets=rule)
            assert torch.equal(g[i, :g1.shape[1]], g1[0])
            b1, blp1 = decode.beam_decode(m, [imgs[i]], START, END, 3, LEN, finalize="backtrack", brackets=rule)
            assert torch.equal(b[i, :, :b1.shape[2]], b1[0]) and torch.equal(blp[i], blp1[0])
            cell, _ = bo.torch_cells(_d(pd), rm.encoder_forward(_d(pe), imgs[i][None].double()).reshape(1, -1, 512), 1, START)
            assert torch.equal(g1, bo.greedy(bo.first(cell), 1, rule, END, LEN + 1))


def test_all_neutral_table_changes_nothing(torch_setup):
    """a table without kinds: ids, log-probs and attention bit for bit those of the call without a rule"""
    from latex_ocr_b200 import decode
    pe, pd, img, _, m = torch_setup
    rule = decode.BracketRule([0] * V)
    a = decode.greedy_decode(m, img, START, END, LEN, return_attention=True)
    b = decode.greedy_decode(m, img, START, END, LEN, return_attention=True, brackets=rule)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    kw = dict(finalize="backtrack", return_attention=True, length_penalty=0.6, coverage_penalty=0.4, return_scores=True)
    a = decode.beam_decode(m, img, START, END, 3, LEN, **kw)
    b = decode.beam_decode(m, img, START, END, 3, LEN, brackets=rule, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    kw = dict(max_length_formula=LEN, seed=4, return_attention=True, top_p=0.9)
    a = decode.sample_decode(m, img, START, END, 4, **kw)
    b = decode.sample_decode(m, img, START, END, 4, brackets=rule, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    dec, enc = _tf_decoder(_tf_p()), _tf_enc(6, 12, 8).cuda()
    a = dec.decode(enc, return_attention=True)
    b = dec.decode(enc, return_attention=True, brackets=decode.BracketRule([0] * TF_V))
    assert torch.equal(a[0].ids, b[0].ids) and torch.equal(a[1], b[1])


def test_reference_finalize_is_refused(torch_setup, ext_setup):
    from latex_ocr_b200 import decode, ext
    _, _, img, _, m = torch_setup
    rule = _rule()
    with pytest.raises(ValueError, match="backtrack"):
        decode.beam_decode(m, img, START, END, 3, LEN, brackets=rule)
    with pytest.raises(ValueError, match="backtrack"):
        ext.beam_decode(ext_setup[3], img, START, END, 3, max_length_formula=LEN, finalize="reference", brackets=rule)
    with pytest.raises(ValueError, match="backtrack"):
        _tf_decoder(_tf_p(), "beam_search", 3).decode(_tf_enc(2, 12, 8).cuda(), brackets=_rule(TF_V))
    with pytest.raises(ValueError, match="END"):
        decode.greedy_decode(m, img, START, OPEN, LEN, brackets=rule)
    closes = decode.BracketRule([0 if v == END else (1 if v == OPEN else -1) for v in range(V)])   # END and { allowed at step 0
    with pytest.raises(ValueError, match="beam_size"):
        decode.beam_decode(m, img, START, END, 3, LEN, finalize="backtrack", brackets=closes)


# ------------------------------------------------------------------------------------------------ trainers
class _Vocab:
    def __init__(self, n):
        self.n_tok = n
        self.id_unk, self.id_pad, self.id_end = n - 3, n - 2, n - 1
        self.id_to_tok = {i: t for i, t in enumerate(_toks(n - 3) + ["_UNK", "_PAD", "_END"])}
        self.tok_to_id = {t: i for i, t in self.id_to_tok.items()}


def _as_ids(vocab, hyps):
    return [[vocab.tok_to_id[t] for t in h.split()] if isinstance(h, str) else list(h) for h in hyps]


@pytest.mark.parametrize("decoding", ["greedy", "beam_search"])
def test_torch_trainer_switch(tmp_path, decoding):
    from latex_ocr_b200.img2seq import Img2SeqModel
    from oracle import ref_model as rm
    vocab = _Vocab(V)
    pe, pd = _torch_params(21)
    rng = np.random.RandomState(0)
    data = [(rng.randint(0, 256, (32, 64, 1)).astype(np.uint8), list(rng.randint(0, V - 3, 3 + i % 3))) for i in range(6)]
    img = [d[0] for d in data]

    def model(on):
        cfg = Cfg(batch_size=3, max_length_formula=LEN, decoding=decoding, beam_size=3, dir_answers=str(tmp_path) + "/a%s/" % on,
                  **({} if on is None else {"balanced_brackets": on}))
        m = Img2SeqModel(cfg, dir_output=str(tmp_path), vocab=vocab, device="cuda", precision="fp32").build_train()
        m.encoder.load_state_dict(pe)
        m.decoder.load_state_dict(pd)
        return m, cfg
    from latex_ocr_b200 import decode
    rule = decode.BracketRule.latex(vocab.id_to_tok)
    m0, _ = model(None)
    free = m0.predict_batch(img)
    _bites(rule, _as_ids(vocab, free[0]))
    m1, cfg1 = model(True)
    for hyps in m1.predict_batch(img) + m1.predict_images(img):
        _ok(rule, _as_ids(vocab, hyps))
    assert np.isfinite(m1.evaluate(cfg1, data)["perplexity"])
    _ok(rule, _as_ids(vocab, open(str(tmp_path) + "/aTrue/hyp_0.txt").read().splitlines()))
    # the switch off: the predictions of a model without it
    m2, _ = model(False)
    assert m2.predict_batch(img) == free and m2.predict_images(img) == m0.predict_images(img)


def test_tf_trainer_switch():
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    vocab = _Vocab(TF_V)
    rng = np.random.RandomState(3)
    data = [(rng.randint(0, 256, (32, 64, 1)).astype(np.uint8), list(rng.randint(0, TF_V - 3, 3 + i % 3))) for i in range(6)]
    p = _tf_params(7)
    for decoding in ("greedy", "beam_search"):
        cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=LEN,
                  decoding=decoding, beam_size=3, batch_size=3, balanced_brackets=True)
        m = Img2SeqModel(cfg, vocab=vocab, device="cuda", precision="fp32", impl="simt").build_train(cfg)
        m.decoder.load_tf_variables(p)
        rule = m._decode_kw()["brackets"]
        for hyps in m.predict_batch([d[0] for d in data]) + m.predict_images([d[0] for d in data]):
            _ok(rule, hyps)
        assert np.isfinite(m.evaluate(cfg, data)["perplexity"])
        cfg.balanced_brackets = False
        assert m._decode_kw() == {}
