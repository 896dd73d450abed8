"""-m gpu: greedy and beam decode of the row-encoder extension (ext.greedy_decode / ext.beam_decode: CNN -> row encoder ->
two-layer decoder in one CUDA time loop, lo_decoder2_greedy / lo_decoder2_beam) against the float64 CPU oracle of
tests/decoder2_decode_oracle.py (oracle/ref_ext.py's model, no dropout).  fp32: ids exact, attention 1e-5, log-probs and scores
1e-3 relative (as the other flavours' decode tests); bf16: a stated token-match rate and run-to-run bit identity.  decode.* on the
same model keeps its layer-1-only path."""
import pytest
import torch

import beam_penalty_oracle as bpo
import decoder2_decode_oracle as d2o
from util import Cfg

pytestmark = pytest.mark.gpu

V = 30
START, END = V - 2, 5
LEN = 8


def _rel(got, want):
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).double()
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())


def _d(p):
    return {k: v.double() for k, v in p.items()}


def _params(seed, V=V):
    from oracle import ref_ext as rx
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    prow, p2 = rx.init_params_ext(seed=seed + 1)
    g = torch.Generator().manual_seed(seed)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    return pe, prow, pd, p2


def _model(params, precision, V=V):
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


@pytest.fixture(scope="module")
def setup():
    from oracle import ref_model as rm
    params = _params(21)
    pe, prow, pd, p2 = params
    img, _ = rm.synthetic_batch(6, 32, 64, V, 3, 5, seed=3)
    enc = d2o.encode(_d(pe), _d(prow), img.double())
    return params, _model(params, "fp32"), img, enc


def test_greedy_fp32_matches_the_oracle(setup):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, img, enc = setup
    want, _, watt = d2o.greedy_decode(_d(pd), _d(p2), enc, START, END, LEN + 1)
    ids, att = ext.greedy_decode(m, img, START, END, LEN, return_attention=True)
    assert torch.equal(ids, want)
    assert att.shape == watt.shape and (att.double() - watt).abs().max().item() < 1e-5
    assert torch.equal(ext.greedy_decode(m, img, START, END, LEN), ids)


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
@pytest.mark.parametrize("beam", [1, 3, 5])
@pytest.mark.parametrize("ab", [(0.0, 0.0), (0.6, 0.4)])
def test_beam_fp32_matches_the_oracle(setup, ab, beam, fin):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, img, enc = setup
    alpha, beta = ab
    want, wlp, wsc = d2o.beam_decode(_d(pd), _d(p2), enc, START, END, beam, LEN + 1, finalize=fin, alpha=alpha, beta=beta)
    ids, lp, sc = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, finalize=fin, length_penalty=alpha,
                                  coverage_penalty=beta, return_scores=True)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3
    ids2, lp2 = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, finalize=fin, length_penalty=alpha,
                                coverage_penalty=beta)
    assert torch.equal(ids2, ids) and torch.equal(lp2, lp)


def test_beam_fp32_with_injected_diversity_uniforms(setup):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, img, enc = setup
    beam = 3
    div = dict(div_gamma=0.5, div_prob=0.7, div_u=torch.rand(LEN + 2, img.shape[0] * beam, V, generator=torch.Generator().manual_seed(77)))
    base, _, _ = d2o.beam_decode(_d(pd), _d(p2), enc, START, END, beam, LEN + 1)
    want, wlp, wsc = d2o.beam_decode(_d(pd), _d(p2), enc, START, END, beam, LEN + 1, alpha=0.6, beta=0.4,
                                     **{k: (v.double() if torch.is_tensor(v) else v) for k, v in div.items()})
    assert want.shape != base.shape or not torch.equal(want, base)
    ids, lp, sc = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, length_penalty=0.6, coverage_penalty=0.4,
                                  return_scores=True, **div)
    assert torch.equal(ids, want.permute(0, 2, 1))
    assert _rel(lp, wlp) < 1e-3 and _rel(sc, wsc) < 1e-3


@pytest.mark.parametrize("fin", ["reference", "backtrack"])
def test_beam_attention_both_views(setup, fin):
    """'reference': the rows slot s computed at each step (the oracle's recorded rows); 'backtrack': the attention under which each
    token of the hypothesis was chosen (the recorded row of its parent at that step)"""
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, img, enc = setup
    beam = 3
    step, reorder, _ = d2o.cell(_d(pd), _d(p2), enc, beam, START)
    rec = []

    def stepped(tok):
        lg, a = step(tok)
        rec.append(a)
        return lg, a
    _, parents, _, _ = bpo.search(stepped, reorder, enc.shape[0], beam, V, END, LEN + 1, dtype=torch.float64)
    ids, lp, att = ext.beam_decode(m, img, START, END, beam, max_length_formula=LEN, finalize=fin, return_attention=True)
    N, n, R = enc.shape[0], len(rec), enc.shape[1]
    assert att.shape == (N, beam, n, R)
    rows = torch.stack(rec).view(n, N, beam, R)                           # [t][i][slot][r]
    for i in range(N):
        for s in range(beam):
            cur = s
            for t in range(n - 1, -1, -1):
                if fin == "reference":
                    w = rows[t, i, s]
                else:
                    p = int(parents[i, t, cur])
                    w = rows[t, i, p]
                    cur = p
                assert (att[i, s, t].double() - w).abs().max().item() < 1e-5, (i, s, t)


def _mixed(seed, shapes=((32, 64), (48, 96), (32, 200), (48, 64)), per=2):
    from oracle import ref_model as rm
    groups = [rm.synthetic_batch(per, H, W, V, 3, 5, seed=seed + k)[0] for k, (H, W) in enumerate(shapes)]
    return [groups[k][i] for i in range(per) for k in range(len(shapes))]


def test_mixed_sizes_match_the_oracle_per_image(setup):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, _, _ = setup
    imgs = _mixed(40)
    ids, att = ext.greedy_decode(m, imgs, START, END, LEN, return_attention=True)
    bids, blp = ext.beam_decode(m, imgs, START, END, 3, max_length_formula=LEN, finalize="backtrack")
    for i, x in enumerate(imgs):
        enc = d2o.encode(_d(pe), _d(prow), x.unsqueeze(0).double())
        want, _, watt = d2o.greedy_decode(_d(pd), _d(p2), enc, START, END, LEN + 1)
        n = want.shape[1]
        assert torch.equal(ids[i, :n], want[0]), i
        assert att[i].shape[1] == enc.shape[1] and (att[i][:n].double() - watt[0]).abs().max().item() < 1e-5, i
        wb, wlp, _ = d2o.beam_decode(_d(pd), _d(p2), enc, START, END, 3, LEN + 1, finalize="backtrack")
        nb = wb.shape[1]
        assert torch.equal(bids[i, :, :nb], wb[0].permute(1, 0)), i
        assert _rel(blp[i], wlp[0]) < 1e-3


def test_uniform_list_equals_the_tensor_path_bit_for_bit(setup):
    from latex_ocr_b200 import ext
    _, m, img, _ = setup
    ids_t, al_t = ext.greedy_decode(m, img, START, END, LEN, return_attention=True)
    ids_l, al_l = ext.greedy_decode(m, list(img), START, END, LEN, return_attention=True)
    assert torch.equal(ids_t, ids_l) and torch.equal(al_t, torch.stack(al_l))
    b_t = ext.beam_decode(m, img, START, END, 5, max_length_formula=LEN, length_penalty=0.6, return_scores=True)
    b_l = ext.beam_decode(m, list(img), START, END, 5, max_length_formula=LEN, length_penalty=0.6, return_scores=True)
    for x, y in zip(b_t, b_l):
        assert torch.equal(x, y)


def test_an_image_decodes_the_same_alone_and_in_any_composition(setup):
    from latex_ocr_b200 import _lib, ext
    _, m, _, _ = setup
    small = _mixed(60, shapes=((32, 64), (48, 160)), per=2)
    big = small + _mixed(70, per=4)
    perm = torch.randperm(len(big), generator=torch.Generator().manual_seed(3)).tolist()
    big = [big[i] for i in perm]
    pos = [perm.index(i) for i in range(len(small))]
    with _lib.option(att_nsplit=3):                       # a fixed split partitions every row alike whatever the composition
        ids_s, al_s = ext.greedy_decode(m, small, START, END, LEN, return_attention=True)
        ids_b, al_b = ext.greedy_decode(m, big, START, END, LEN, return_attention=True)
        bs, lps = ext.beam_decode(m, small, START, END, 3, max_length_formula=LEN)
        bb, lpb = ext.beam_decode(m, big, START, END, 3, max_length_formula=LEN)
    n = ids_s.shape[1]
    assert torch.equal(ids_s, ids_b[pos, :n])
    for i, p in enumerate(pos):
        assert torch.equal(al_s[i], al_b[p][:n])
    nb = bs.shape[2]
    assert torch.equal(bs, bb[pos, :, :nb]) and torch.equal(lps, lpb[pos])


def test_above_1024_rows(setup):
    """206 images x beam 5 = 1030 rows (six distinct images repeated): every image gets its source's oracle hypotheses"""
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), m, img, enc = setup
    reps = 206 // img.shape[0] + 1
    big = img.repeat(reps, 1, 1, 1)[:206]
    want, wlp, _ = d2o.beam_decode(_d(pd), _d(p2), enc, START, END, 5, LEN + 1)
    ids, lp = ext.beam_decode(m, big, START, END, 5, max_length_formula=LEN)
    src = torch.arange(206) % img.shape[0]
    assert torch.equal(ids, want.permute(0, 2, 1)[src])
    assert _rel(lp, wlp[src]) < 1e-3


def test_bf16_at_cfg4_size_token_match_and_bit_identity():
    """160 x 640 images (cfg4), V = 500, bf16 on the tensor-core kernels: the tokens agree with the float64 oracle on the same
    bf16-rounded weights at a STATED rate >= 0.9 (greedy, over each row's tokens up to the oracle's first END), and two runs of
    greedy and beam 5 are bit-identical."""
    from latex_ocr_b200 import ext
    from oracle import ref_model as rm
    Vc, n_img, L = 500, 4, 30
    params = _params(31, Vc)
    params = tuple({k: (v.bfloat16().float() if v.dim() >= 2 else v) for k, v in p.items()} for p in params)
    m = _model(params, "bf16", Vc)
    img, _ = rm.synthetic_batch(n_img, 160, 640, Vc, 3, 5, seed=9)
    g1 = ext.greedy_decode(m, img, Vc - 2, Vc - 1, L)
    b1 = ext.beam_decode(m, img, Vc - 2, Vc - 1, 5, max_length_formula=L, return_scores=True, length_penalty=0.6)
    g2 = ext.greedy_decode(m, img, Vc - 2, Vc - 1, L)
    b2 = ext.beam_decode(m, img, Vc - 2, Vc - 1, 5, max_length_formula=L, return_scores=True, length_penalty=0.6)
    assert torch.equal(g1, g2) and all(torch.equal(x, y) for x, y in zip(b1, b2))
    pe, prow, pd, p2 = params
    enc = d2o.encode(_d(pe), _d(prow), img.double())
    want, _, _ = d2o.greedy_decode(_d(pd), _d(p2), enc, Vc - 2, Vc - 1, L + 1)
    hit = tot = 0
    for i in range(n_img):
        w = want[i].tolist()
        n = w.index(Vc - 1) + 1 if Vc - 1 in w else len(w)
        hit += sum(int(a == b) for a, b in zip(g1[i, :n].tolist(), w[:n]))
        tot += n
    rate = hit / tot
    print("bf16 cfg4 greedy token match vs float64 oracle: %.3f over %d tokens" % (rate, tot))
    assert rate >= 0.9, rate


def test_decode_module_keeps_the_layer1_path(setup):
    """decode.greedy_decode / beam_decode on the row model still run encoder -> decoder (no row encoder, no layer 2): exactly what
    the one-layer Img2SeqModel with the same CNN and decoder weights returns"""
    from latex_ocr_b200 import decode, ext
    from util import build_model
    (pe, prow, pd, p2), m, img, _ = setup
    one = build_model(V, pe, pd, "fp32")
    ids, att = decode.greedy_decode(m, img, START, END, LEN, return_attention=True)
    ids1, att1 = decode.greedy_decode(one, img, START, END, LEN, return_attention=True)
    assert torch.equal(ids, ids1) and torch.equal(att, att1)
    b = decode.beam_decode(m, img, START, END, 3, LEN, length_penalty=0.6, return_scores=True)
    b1 = decode.beam_decode(one, img, START, END, 3, LEN, length_penalty=0.6, return_scores=True)
    assert all(torch.equal(x, y) for x, y in zip(b, b1))
    ext.greedy_decode(m, img, START, END, LEN)                     # the two-layer decode leaves the one-layer path as it was
    assert torch.equal(decode.greedy_decode(m, img, START, END, LEN), ids)
