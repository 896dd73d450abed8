"""-m gpu: sampling decode in the three decoder flavours (decode.sample_decode / lo_decoder_sample, tf_decoder.Decoder.sample /
lo_tfdec_sample, ext.sample_decode / lo_decoder2_sample) against the float64 restatement of tests/sample_oracle.py on the
oracles' own cells, and decode.mbr_select against a CPU Levenshtein.

fp32 with injected uniforms: ids equal and log-probs within 1e-5 (relative to max(1, |log-prob|)).  The top-p values are chosen
per case from a fixed list so that every draw's token masses lie at least 1e-4 from p (the oracle reports that margin), so the
fp32 rounding of the masses cannot change a kept set."""
import numpy as np
import pytest
import torch

import sample_oracle as so
from latex_ocr_b200 import _lib, decode, philox
from test_gpu_beam_penalty import _params as _torch_params, _tf_enc, _tf_params
from test_gpu_ext_decode import _d, _model as _ext_model, _params as _ext_params
from test_sample_abi import _mbr_rule
from util import Cfg, build_model

pytestmark = pytest.mark.gpu

V, TF_V = 30, 40
START, END = V - 2, 5
LEN = 8
N_S = 4
P_CANDIDATES = (0.9, 0.8, 0.7, 0.85, 0.75, 0.95, 0.6, 0.65)
SETTINGS = [(1.0, 0, 1.0), (0.7, 5, 1.0), (1.3, 0, None), (1.0, 8, None)]     # (tau, top_k, top_p); None: chosen by margin


def _rel(got, want):
    got, want = torch.as_tensor(got).cpu().double(), torch.as_tensor(want).double()
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())


def _u(steps, B, Vv, seed):
    return torch.rand(steps, B, Vv, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).clamp_(1e-6, 1 - 1e-6).float()


def _oracle(make_cell, tau, k, p, u, max_iter=LEN + 1):
    """(top_p, ids [B, steps], log-probs [B]) of the oracle; p None: the first candidate whose margin is >= 1e-4"""
    for pp in ((p,) if p is not None else P_CANDIDATES):
        cell, B = make_cell()
        ids, lp, margin = so.search(cell, B, END, max_iter, tau, k, pp, u)
        if margin >= 1e-4:
            return pp, ids, lp
    raise AssertionError("no top-p candidate keeps every mass 1e-4 from p")


def _check(ids, lp, want, wlp):
    N, n, steps = ids.shape
    assert torch.equal(ids.reshape(N * n, steps), want)
    err = _rel(lp.reshape(-1), wlp)
    print("log-prob error %.2e" % err)
    assert err < 1e-5


# ------------------------------------------------------------------------------------------------ the three flavours
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


def _tf_decoder(p, precision="fp32"):
    from latex_ocr_b200.tf_decoder import Decoder
    cfg = Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=LEN)
    dec = Decoder(cfg, TF_V, END, device="cuda", precision=precision, impl="simt" if precision == "fp32" else "tc")
    dec.load_tf_variables(p)
    return dec


@pytest.mark.parametrize("tau,k,p", SETTINGS)
def test_torch_matches_the_oracle(torch_setup, tau, k, p):
    pe, pd, img, enc, m = torch_setup
    u = _u(LEN + 2, img.shape[0] * N_S, V, 11)
    p, want, wlp = _oracle(lambda: so.torch_cell(_d(pd), enc, N_S, START), tau, k, p, u)
    ids, lp = decode.sample_decode(m, img, START, END, N_S, tau, k, p, LEN, u=u)
    _check(ids, lp, want, wlp)


@pytest.mark.parametrize("tau,k,p", SETTINGS)
def test_tf_matches_the_oracle(tau, k, p):
    tp = _tf_params(7)
    enc = _tf_enc(6, 12, 8)
    u = _u(LEN + 2, 6 * N_S, TF_V, 12)
    p, want, wlp = _oracle(lambda: so.tf_cell(_d(tp), enc.double(), N_S), tau, k, p, u)
    ids, lp = _tf_decoder(tp).sample(enc.cuda(), N_S, tau, k, p, u=u)
    _check(ids.cpu(), lp.cpu(), want, wlp)


@pytest.mark.parametrize("tau,k,p", SETTINGS)
def test_decoder2_matches_the_oracle(ext_setup, tau, k, p):
    from latex_ocr_b200 import ext
    (pe, prow, pd, p2), img, enc, m = ext_setup
    u = _u(LEN + 2, img.shape[0] * N_S, V, 13)
    p, want, wlp = _oracle(lambda: so.decoder2_cell(_d(pd), _d(p2), enc, N_S, START), tau, k, p, u)
    ids, lp = ext.sample_decode(m, img, START, END, N_S, temperature=tau, top_k=k, top_p=p, max_length_formula=LEN, u=u)
    _check(ids, lp, want, wlp)


def _through_end(greedy, n):
    """greedy ids [N, steps] -> [N, n, steps] with every position after the first END set to END (a sample emits END then)"""
    g = greedy.clone()
    for row in g:
        hit = (row == END).nonzero()
        if hit.numel():
            row[int(hit[0]) + 1:] = END
    return g.unsqueeze(1).expand(-1, n, -1)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_top_k_1_is_greedy_decode(torch_setup, ext_setup, precision):
    from latex_ocr_b200 import ext
    pe, pd, img, _, _ = torch_setup
    m = build_model(V, pe, pd, precision, impl="tc" if precision == "bf16" else "simt")
    g = decode.greedy_decode(m, img, START, END, LEN)
    ids, _ = decode.sample_decode(m, img, START, END, 3, 1.7, 1, 1.0, LEN, seed=1)
    assert torch.equal(ids, _through_end(g, 3))
    params, img2, _, _ = ext_setup
    m2 = _ext_model(params, precision)
    g = ext.greedy_decode(m2, img2, START, END, LEN)
    ids, _ = ext.sample_decode(m2, img2, START, END, 3, temperature=0.6, top_k=1, max_length_formula=LEN, seed=2)
    assert torch.equal(ids, _through_end(g, 3))
    dec = _tf_decoder(_tf_params(7), precision)
    enc = _tf_enc(6, 12, 8).cuda()
    g = dec.decode(enc).ids
    ids, _ = dec.sample(enc, 3, 1.2, 1, 0.5, seed=3)
    assert torch.equal(ids.cpu(), _through_end(g.cpu(), 3))


# ------------------------------------------------------------------------------------------------ Philox
def test_philox_draws_reproduce_and_match_the_host_mirror(torch_setup):
    pe, pd, img, enc, m = torch_setup
    m16 = build_model(V, pe, pd, "bf16", impl="tc")
    a = decode.sample_decode(m16, img, START, END, N_S, 1.0, 0, 1.0, LEN, seed=5)
    b = decode.sample_decode(m16, img, START, END, N_S, 1.0, 0, 1.0, LEN, seed=5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = decode.sample_decode(m16, img, START, END, N_S, 1.0, 0, 1.0, LEN, seed=6)
    assert not torch.equal(a[0], c[0])
    d = decode.sample_decode(m16, img, START, END, N_S, 1.0, 0, 1.0, LEN)
    e = decode.sample_decode(m16, img, START, END, N_S, 1.0, 0, 1.0, LEN)
    assert not torch.equal(d[0], e[0]) and int(m16._sample_state[1]) == 2
    # fp32: the kernel's Philox uniforms are the host mirror's
    B = img.shape[0] * N_S
    u = torch.from_numpy(philox.gumbel_uniforms(4242, 0, B, LEN + 2, V)).permute(1, 0, 2).contiguous()
    _, want, wlp = _oracle(lambda: so.torch_cell(_d(pd), enc, N_S, START), 0.9, 0, 1.0, u)
    ids, lp = decode.sample_decode(m, img, START, END, N_S, 0.9, 0, 1.0, LEN, seed=4242)
    _check(ids, lp, want, wlp)


# ------------------------------------------------------------------------------------------------ distribution
def test_draws_follow_the_filtered_softmax(torch_setup):
    """fc.weight = 0, fc.bias = fixed logits: every step draws from the filtered softmax(bias / tau); END is filtered out, so no
    row ends and every step of every row is one draw"""
    from scipy.stats import chisquare
    pe, pd, _, _, _ = torch_setup
    from oracle import ref_model as rm
    bias = torch.linspace(-1.5, 1.0, V)
    pd = dict(pd, **{"fc.weight": torch.zeros_like(pd["fc.weight"]), "fc.bias": bias})
    m = build_model(V, pe, pd, "fp32")
    img, _ = rm.synthetic_batch(64, 32, 64, V, 3, 5, seed=8)
    tau, k, p = 1.5, 12, 0.5
    kept, margin = so.keep_mask(bias.double().numpy(), tau, k, p)
    assert margin > 1e-4 and not kept[END] and 2 < kept.sum() < k
    counts = np.zeros(V)
    for call in range(3):
        ids, _ = decode.sample_decode(m, img, START, END, 16, tau, k, p, LEN)
        assert ids.shape == (64, 16, LEN + 2)
        counts += np.bincount(ids.reshape(-1).numpy(), minlength=V)
    assert counts[~kept].sum() == 0                      # filtered-out tokens are never drawn
    q = np.exp(bias.double().numpy() / tau)
    q = np.where(kept, q, 0.0)
    q /= q.sum()
    stat, pval = chisquare(counts[kept], q[kept] * counts.sum())
    print("chi-square %.2f over %d draws, %d tokens kept, p = %.3f" % (stat, counts.sum(), kept.sum(), pval))
    assert pval > 1e-3


# ------------------------------------------------------------------------------------------------ sizes
def test_mixed_sizes_each_image_as_alone(torch_setup):
    from oracle import ref_model as rm
    pe, pd, _, _, m = torch_setup
    shapes = ((32, 64), (48, 96), (32, 200), (48, 64), (32, 128))
    groups = [rm.synthetic_batch(2, H, W, V, 3, 5, seed=40 + k)[0] for k, (H, W) in enumerate(shapes)]
    imgs = [groups[k][i] for i in range(2) for k in range(len(shapes))]
    n = 3
    u = _u(LEN + 2, len(imgs) * n, V, 21)
    kw = dict(n_samples=n, temperature=1.1, top_k=10, top_p=0.95, max_length_formula=LEN)
    with _lib.option(att_nsplit=3):                       # a fixed split partitions every row alike whatever the composition
        ids, lp, att = decode.sample_decode(m, imgs, START, END, u=u, return_attention=True, **kw)
        assert len(att) == len(imgs)
        for i in (0, 3, 7, 9):
            ids_a, lp_a = decode.sample_decode(m, [imgs[i]], START, END, u=u[:, i * n:(i + 1) * n].clone(), **kw)
            s = ids_a.shape[2]
            assert torch.equal(ids[i, :, :s], ids_a[0]) and (ids[i, :, s:] == END).all()
            assert torch.equal(lp[i], lp_a[0])
            assert att[i].shape[:2] == (n, ids.shape[2])
        # the reversed composition
        rev = imgs[::-1]
        ur = u.view(LEN + 2, len(imgs), n, V).flip(1).reshape(LEN + 2, len(imgs) * n, V)
        ids_r, lp_r = decode.sample_decode(m, rev, START, END, u=ur, **kw)
        assert torch.equal(ids_r.flip(0), ids) and torch.equal(lp_r.flip(0), lp)


def test_tf_mixed_sizes_each_image_as_alone():
    tp = _tf_params(7)
    dec = _tf_decoder(tp)
    encs = [_tf_enc(1, R, 30 + R)[0].cuda() for R in (12, 5, 20, 9)]
    n = 3
    u = _u(LEN + 2, len(encs) * n, TF_V, 22)
    with _lib.option(att_nsplit=3):
        ids, lp = dec.sample(encs, n, 1.0, 7, 1.0, u=u)
        for i, e in enumerate(encs):
            ids_a, lp_a = dec.sample([e], n, 1.0, 7, 1.0, u=u[:, i * n:(i + 1) * n].clone())
            s = ids_a.shape[2]
            assert torch.equal(ids[i, :, :s], ids_a[0]) and (ids[i, :, s:] == END).all()
            assert torch.equal(lp[i], lp_a[0])


def test_more_than_1024_rows(torch_setup):
    """128 images x 9 samples = 1,152 rows in one call equal the same images in calls of 16"""
    from oracle import ref_model as rm
    pe, pd, _, _, m = torch_setup
    img, _ = rm.synthetic_batch(128, 32, 64, V, 3, 5, seed=17)
    n = 9
    u = _u(LEN + 2, 128 * n, V, 23)
    kw = dict(n_samples=n, temperature=1.0, top_k=0, top_p=0.9, max_length_formula=LEN)
    with _lib.option(att_nsplit=3):
        ids, lp = decode.sample_decode(m, img, START, END, u=u, **kw)
        for c in range(0, 128, 16):
            ids_c, lp_c = decode.sample_decode(m, img[c:c + 16], START, END, u=u[:, c * n:(c + 16) * n].clone(), **kw)
            s = ids_c.shape[2]
            assert torch.equal(ids[c:c + 16, :, :s], ids_c) and (ids[c:c + 16, :, s:] == END).all()
            assert torch.equal(lp[c:c + 16], lp_c)


# ------------------------------------------------------------------------------------------------ MBR
def test_mbr_select_matches_a_cpu_levenshtein(torch_setup):
    pe, pd, img, _, _ = torch_setup
    m16 = build_model(V, pe, pd, "bf16", impl="tc")
    ids, _ = decode.sample_decode(m16, img, START, END, 8, 1.5, 0, 1.0, LEN, seed=9)
    choice, agree = decode.mbr_select(ids, END)
    means = _mbr_rule(ids, END)
    assert choice.shape == (img.shape[0],) and agree.dtype == torch.float32
    for i, row in enumerate(means):
        best = max(row)
        assert abs(agree[i].item() - best) < 1e-6
        top = sorted(row, reverse=True)
        if top[0] - top[1] > 1e-6:
            assert choice[i].item() == row.index(best)
        else:
            assert abs(row[choice[i].item()] - best) <= 1e-6
            assert choice[i].item() == min(j for j, v in enumerate(row) if best - v <= 1e-6)
    assert len({tuple(r.tolist()) for r in ids[0]}) > 1      # the samples differ
