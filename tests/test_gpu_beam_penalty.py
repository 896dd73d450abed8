"""-m gpu: the length and coverage penalties of beam search (lo_beam_penalty) in both decoder flavours, against the penalised CPU
search of tests/beam_penalty_oracle.py on the oracles' own cells.

The models are random-init with END made likely (so that hypotheses end at different lengths and the length penalty has something
to rank) and sharpened attention (so that hypotheses differ in what they cover), over 12 regions: the coverage term grows with the
region count, and a large term leaves fp32 scores too coarse to rank candidates alike on the device and on the CPU.  Every oracle
case at beam 3 and 5 first checks that its penalties change the search at those settings.  At beam 1 the penalties can only move
END against the best other token (the coverage term is the same for every candidate of the one row): the torch-flavour model's
length penalty does, elsewhere the scores must at least differ from the log-probs."""
import pytest
import torch

import beam_penalty_oracle as bpo
from util import Cfg, build_model

pytestmark = pytest.mark.gpu

V = 30
START, END = V - 2, 5
LEN = 8
PAIRS = [(0.6, 0.0), (0.0, 0.4), (0.6, 0.4), (1.5, 1.0)]


def _rel(got, want):
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).double()
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())


def _check_change(base, pen_ref, lp, sc, must_change):
    """base / pen_ref: the oracle's reference-finalize ids [N, steps, beam] without / with the penalties"""
    if must_change:
        assert pen_ref.shape != base.shape or not torch.equal(pen_ref, base)   # the penalties change the search at these settings
    else:
        assert not torch.equal(sc, lp)


# ------------------------------------------------------------------------------------------------ torch flavour
def _params(seed):
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    pd["fc.bias"][END] += 1.0
    pd["attention.full_att.weight"] *= 10.0
    return pe, pd


def _enc(pe, img):
    from oracle import ref_model as rm
    return rm.encoder_forward(pe, img).reshape(img.shape[0], -1, 512)


@pytest.fixture(scope="module")
def torch_setup():
    from oracle import ref_model as rm
    pe, pd = _params(21)
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=3)
    return pe, pd, build_model(V, pe, pd, "fp32"), img, _enc(pe, img)


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
@pytest.mark.parametrize("beam", [1, 3, 5])
@pytest.mark.parametrize("ab", PAIRS)
def test_torch_matches_the_oracle(torch_setup, ab, beam, fin):
    from latex_ocr_b200 import decode
    alpha, beta = ab
    pe, pd, m, img, enc = torch_setup
    base, _, _ = bpo.beam_decode(pd, enc, START, END, beam, LEN + 1)
    want, wlp, wsc = bpo.beam_decode(pd, enc, START, END, beam, LEN + 1, finalize=fin, alpha=alpha, beta=beta)
    pen_ref = want if fin == "reference" else bpo.beam_decode(pd, enc, START, END, beam, LEN + 1, alpha=alpha, beta=beta)[0]
    _check_change(base, pen_ref, wlp, wsc, beam > 1 or alpha != 0)
    ids, lp, sc = decode.beam_decode(m, img, START, END, beam, LEN, finalize=fin, length_penalty=alpha, coverage_penalty=beta,
                                     return_scores=True)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3
    # the same search without the scores output
    ids2, lp2 = decode.beam_decode(m, img, START, END, beam, LEN, finalize=fin, length_penalty=alpha, coverage_penalty=beta)
    assert torch.equal(ids2, ids) and torch.equal(lp2, lp)


def test_torch_with_injected_diversity_uniforms(torch_setup):
    from latex_ocr_b200 import decode
    pe, pd, m, img, enc = torch_setup
    beam, alpha, beta = 3, 0.6, 0.4
    div = dict(div_gamma=0.5, div_prob=0.7, div_u=torch.rand(LEN + 2, img.shape[0] * beam, V, generator=torch.Generator().manual_seed(77)))
    base, _, _ = bpo.beam_decode(pd, enc, START, END, beam, LEN + 1, **div)
    want, wlp, wsc = bpo.beam_decode(pd, enc, START, END, beam, LEN + 1, alpha=alpha, beta=beta, **div)
    assert want.shape != base.shape or not torch.equal(want, base)
    ids, lp, sc = decode.beam_decode(m, img, START, END, beam, LEN, length_penalty=alpha, coverage_penalty=beta, return_scores=True,
                                     **div)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
def test_torch_list_of_sizes(torch_setup, fin):
    """images of different sizes in one call: every image's ids, log-probs and scores are those it gets decoded alone (the
    coverage is summed over its own regions only) and its ids the oracle's; return_attention comes along unchanged"""
    from latex_ocr_b200 import _lib, decode
    from oracle import ref_model as rm
    pe, pd, m, _, _ = torch_setup
    shapes = ((32, 64), (48, 96), (32, 200), (48, 64), (32, 128))
    groups = [rm.synthetic_batch(2, H, W, V, 3, 5, seed=40 + k)[0] for k, (H, W) in enumerate(shapes)]
    imgs = [groups[k][i] for i in range(2) for k in range(len(shapes))]
    kw = dict(finalize=fin, length_penalty=0.6, coverage_penalty=0.4, return_scores=True)
    with _lib.option(att_nsplit=3):                       # a fixed split partitions every row alike whatever the composition
        ids, lp, sc, att = decode.beam_decode(m, imgs, START, END, 5, LEN, return_attention=True, **kw)
        ids0, lp0, sc0 = decode.beam_decode(m, imgs, START, END, 5, LEN, **kw)
        assert torch.equal(ids, ids0) and torch.equal(lp, lp0) and torch.equal(sc, sc0)
        for i in (0, 3, 7):
            x = imgs[i]
            ids_a, lp_a, sc_a = decode.beam_decode(m, [x], START, END, 5, LEN, **kw)
            n = ids_a.shape[2]
            assert torch.equal(ids[i, :, :n], ids_a[0])
            assert (ids[i, :, n:] == END).all()
            assert torch.equal(lp[i], lp_a[0]) and torch.equal(sc[i], sc_a[0])
            want, wlp, wsc = bpo.beam_decode(pd, _enc(pe, x.unsqueeze(0)), START, END, 5, LEN + 1, finalize=fin, alpha=0.6, beta=0.4)
            assert torch.equal(ids_a, want.permute(0, 2, 1))
            assert _rel(lp_a, wlp) < 1e-3 and _rel(sc_a, wsc) < 1e-3


def test_torch_zero_penalties_are_the_div_entry_point(torch_setup):
    """length_penalty = coverage_penalty = 0 with return_scores runs lo_decoder_beam_pen: the search of lo_decoder_beam_div bit for
    bit (ids of both finalize modes, so the parents too; the steps run, so the finished flags; the log-probs), scores == log-probs;
    dense and a list of sizes"""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    _, _, m, img, _ = torch_setup
    mixed = [rm.synthetic_batch(1, H, W, V, 3, 5, seed=60 + k)[0][0] for k, (H, W) in enumerate(((32, 64), (48, 96), (32, 200)))]
    for x in (img, mixed):
        for fin in ("reference", "backtrack"):
            ids0, lp0 = decode.beam_decode(m, x, START, END, 5, LEN, finalize=fin, div_gamma=0.5, div_prob=0.5, div_seed=3)
            ids, lp, sc = decode.beam_decode(m, x, START, END, 5, LEN, finalize=fin, div_gamma=0.5, div_prob=0.5, div_seed=3,
                                             return_scores=True)
            assert torch.equal(ids, ids0) and torch.equal(lp, lp0) and torch.equal(sc, lp)


def test_torch_bf16_runs_and_is_reproducible(torch_setup):
    from latex_ocr_b200 import decode
    pe, pd, _, img, _ = torch_setup
    m16 = build_model(V, pe, pd, "bf16", impl="tc")
    kw = dict(length_penalty=0.6, coverage_penalty=0.4, return_scores=True)
    for fin in ("reference", "backtrack"):
        a = decode.beam_decode(m16, img, START, END, 5, LEN, finalize=fin, **kw)
        b = decode.beam_decode(m16, img, START, END, 5, LEN, finalize=fin, **kw)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        assert torch.isfinite(a[2]).all() and (a[2] <= 0).all()


# ------------------------------------------------------------------------------------------------ TensorFlow flavour
TF_V = 40
TF_LEN = 10


def _tf_params(seed):
    from oracle import ref_tf_model as tfm
    p = tfm.init_params_tf(TF_V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0
    p["y_W_o"][:, END] += 0.3
    p["att_beta"] = p["att_beta"] * 3.0
    return p


def _tf_decoder(p, beam, alpha, beta, precision="fp32"):
    from latex_ocr_b200.tf_decoder import Decoder
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=TF_LEN,
              decoding="beam_search", beam_size=beam, length_penalty=alpha, coverage_penalty=beta)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision=precision, impl="simt" if precision == "fp32" else "tc")
    dec.load_tf_variables(p)
    return dec


def _tf_enc(N, R, seed):
    return torch.relu(torch.randn(N, R, 512, generator=torch.Generator().manual_seed(seed))) * 0.7


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
@pytest.mark.parametrize("beam", [1, 3, 5])
@pytest.mark.parametrize("ab", PAIRS)
def test_tf_matches_the_oracle(ab, beam, fin):
    alpha, beta = ab
    p = _tf_params(7)
    enc = _tf_enc(6, 12, 8)
    base, _, _ = bpo.tf_beam_decode(p, enc, END, beam, TF_LEN + 1)
    want, wlp, wsc = bpo.tf_beam_decode(p, enc, END, beam, TF_LEN + 1, finalize=fin, alpha=alpha, beta=beta)
    pen_ref = want if fin == "reference" else bpo.tf_beam_decode(p, enc, END, beam, TF_LEN + 1, alpha=alpha, beta=beta)[0]
    _check_change(base, pen_ref, wlp, wsc, beam > 1)
    dec = _tf_decoder(p, beam, alpha, beta)
    out, lp, sc = dec.decode(enc.cuda(), return_log_probs=True, return_scores=True, finalize=fin)
    assert torch.equal(out.ids.cpu(), want)
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3


def test_tf_with_injected_diversity_uniforms():
    p = _tf_params(7)
    enc = _tf_enc(6, 12, 8)
    beam, alpha, beta = 3, 0.6, 0.4
    u = torch.rand(TF_LEN + 2, 6 * beam, TF_V, generator=torch.Generator().manual_seed(78))
    div = dict(div_gamma=0.5, div_prob=0.7, div_u=u)
    base, _, _ = bpo.tf_beam_decode(p, enc, END, beam, TF_LEN + 1, **div)
    want, wlp, wsc = bpo.tf_beam_decode(p, enc, END, beam, TF_LEN + 1, alpha=alpha, beta=beta, **div)
    assert want.shape != base.shape or not torch.equal(want, base)
    from latex_ocr_b200.tf_decoder import Decoder
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=TF_LEN,
              decoding="beam_search", beam_size=beam, length_penalty=alpha, coverage_penalty=beta, div_gamma=0.5, div_prob=0.7)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision="fp32", impl="simt")
    dec.load_tf_variables(p)
    out, lp, sc = dec.decode(enc.cuda(), div_u=u, return_log_probs=True, return_scores=True)
    assert torch.equal(out.ids.cpu(), want)
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
def test_tf_list_of_sizes(fin):
    from latex_ocr_b200 import _lib
    p = _tf_params(9)
    dec = _tf_decoder(p, 5, 0.6, 0.4)
    g = torch.Generator().manual_seed(24)
    shapes = ((3, 4), (2, 5), (2, 6), (2, 4), (3, 3))
    encs = [torch.relu(torch.randn(h * w, 512, generator=g)) * 0.7 for _ in range(2) for h, w in shapes]
    with _lib.option(att_nsplit=3):
        out, lp, sc, att = dec.decode([e.cuda() for e in encs], return_log_probs=True, return_scores=True, return_attention=True,
                                      finalize=fin)
        out0, lp0, sc0 = dec.decode([e.cuda() for e in encs], return_log_probs=True, return_scores=True, finalize=fin)
        assert torch.equal(out.ids, out0.ids) and torch.equal(lp, lp0) and torch.equal(sc, sc0)
        for i in (0, 2, 6):
            e = encs[i]
            out_a, lp_a, sc_a = dec.decode([e.cuda()], return_log_probs=True, return_scores=True, finalize=fin)
            n = out_a.ids.shape[1]
            assert torch.equal(out.ids[i, :n], out_a.ids[0])
            assert torch.equal(lp[i], lp_a[0]) and torch.equal(sc[i], sc_a[0])
            want, wlp, wsc = bpo.tf_beam_decode(p, e[None], END, 5, TF_LEN + 1, finalize=fin, alpha=0.6, beta=0.4)
            assert torch.equal(out_a.ids.cpu(), want)
            assert _rel(lp_a, wlp) < 1e-3 and _rel(sc_a, wsc) < 1e-3


def test_tf_zero_penalties_are_the_div_entry_point():
    p = _tf_params(11)
    dec = _tf_decoder(p, 5, 0.0, 0.0)
    enc = _tf_enc(8, 96, 12).cuda()
    g = torch.Generator().manual_seed(13)
    mixed = [(torch.relu(torch.randn(n, 512, generator=g)) * 0.7).cuda() for n in (32, 96, 50)]
    for x in (enc, mixed):
        for fin in ("reference", "backtrack"):
            out0, lp0 = dec.decode(x, return_log_probs=True, finalize=fin)
            out, lp, sc = dec.decode(x, return_log_probs=True, return_scores=True, finalize=fin)
            assert torch.equal(out.ids, out0.ids) and torch.equal(lp, lp0) and torch.equal(sc, lp)


def test_tf_bf16_runs_and_is_reproducible():
    p = _tf_params(11)
    dec = _tf_decoder(p, 5, 0.6, 0.4, precision="bf16")
    enc = _tf_enc(40, 96, 12).cuda()
    for fin in ("reference", "backtrack"):
        out_a, lp_a, sc_a = dec.decode(enc, return_log_probs=True, return_scores=True, finalize=fin)
        out_b, lp_b, sc_b = dec.decode(enc, return_log_probs=True, return_scores=True, finalize=fin)
        assert torch.equal(out_a.ids, out_b.ids) and torch.equal(lp_a, lp_b) and torch.equal(sc_a, sc_b)
        assert torch.isfinite(sc_a).all()


def test_model_config_keys_reach_the_search(torch_setup):
    """Img2SeqModel reads length_penalty / coverage_penalty from its config: predict_batch ranks by them"""
    from latex_ocr_b200 import decode
    _, _, m, img, _ = torch_setup
    cfg = m._config
    saved = {k: getattr(cfg, k, None) for k in ("decoding", "beam_size", "max_length_formula", "length_penalty", "coverage_penalty")}
    try:
        cfg.decoding, cfg.beam_size, cfg.max_length_formula = "beam_search", 5, LEN
        cfg.length_penalty, cfg.coverage_penalty = 0.6, 0.4
        got, _ = m._decode_ids(img, start_id=START)
        ids, _ = decode.beam_decode(m, img, START, m._end_id(), 5, LEN, length_penalty=0.6, coverage_penalty=0.4)
        assert got == [ids[:, k].tolist() for k in range(5)]
        cfg.length_penalty = -1.0
        with pytest.raises(ValueError):
            m._decode_ids(img, start_id=START)
    finally:
        for k, v in saved.items():
            if v is None:
                cfg.__dict__.pop(k, None)
            else:
                setattr(cfg, k, v)
