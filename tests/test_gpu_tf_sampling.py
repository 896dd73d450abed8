"""-m gpu: scheduled sampling and self-critical training on the TensorFlow-flavour decoder — the token choice inside the CUDA time
loop (tf_decoder.Decoder.train_outputs(..., sampling_prob, sampling_temperature)), the TF-layout reward and policy gradient
(scst.rewards(..., layout="tf"), scst.pg_grad_tf), and img2seq_tf.Img2SeqModel's set_sampling_prob / set_self_critical.  TF dims of
configs/model.json; oracle: oracle/ref_tf_model.py under float64 autograd."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from latex_ocr_b200 import _lib, metrics, philox, scst
from test_gpu_tf_autograd import _cfg, _keeps, _setup, _tf_batch, _tf_model, custom_loss
from util import relerr

pytestmark = pytest.mark.gpu

PRECISIONS = [("fp32", "simt"), ("bf16", "tc")]


def _run(dec, enc, formula, p, tau=0.0, kh=None, ko=None):
    with torch.no_grad():
        logits, alphas = dec.train_outputs(enc.cuda(), formula.cuda(), kh, ko, sampling_prob=p, sampling_temperature=tau)
    return logits, alphas, dec.last_fed_tokens.clone()


def _check_argmax_rule(logits, fed, formula, u, p):
    want = torch.where(torch.as_tensor(u).cuda() < p, logits.argmax(dim=-1), formula.cuda())
    assert torch.equal(fed, want)


# 1 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [28, 868])
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_argmax_rule_injected_and_philox(precision, impl, R):
    tfm, p, dec, enc, formula = _setup(V=40, N=5, R=R, T=9, seed=31, precision=precision, impl=impl)
    N, T = formula.shape
    u = torch.rand(N, T, generator=torch.Generator().manual_seed(2))
    dec._ss_u = u.cuda()
    logits, _, fed = _run(dec, enc, formula, 0.5)
    _check_argmax_rule(logits, fed, formula, u, 0.5)
    assert (fed != formula.cuda()).any() and (fed == formula.cuda()).any()
    dec._ss_u = None
    dec.seed_sampling(1234, call=7)
    logits, _, fed = _run(dec, enc, formula, 0.5)
    _check_argmax_rule(logits, fed, formula, philox.sampling_uniforms(1234, 7, N, T), 0.5)
    assert int(dec.ss_state[1]) == 8


def _check_draws(logits, fed, u, tau):
    """fed[b][t] = argmax(logits[b][t] / tau - log(-log u)) in float64 where the top-2 gap exceeds 1e-4, one of the two elsewhere"""
    s = logits.double().cpu() / tau - torch.log(-torch.log(torch.as_tensor(u).double()))
    top = torch.topk(s, 2, dim=-1)
    gap = top.values[..., 0] - top.values[..., 1]
    fed = fed.cpu()
    sure = gap > 1e-4
    assert torch.equal(fed[sure], top.indices[..., 0][sure])
    assert ((fed == top.indices[..., 0]) | (fed == top.indices[..., 1])).all()
    assert sure.sum() > 0.9 * sure.numel()


@pytest.mark.parametrize("R", [28, 868])
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_gumbel_rule_injected_and_philox(precision, impl, R):
    V = 40
    tfm, p, dec, enc, formula = _setup(V=V, N=5, R=R, T=9, seed=33, precision=precision, impl=impl)
    N, T = formula.shape
    u = torch.rand(N, T, V, generator=torch.Generator().manual_seed(3)).clamp_(1e-6, 1 - 1e-6)
    for tau in (0.5, 1.0, 2.0):
        dec._ss_gu = u.cuda()
        logits, _, fed = _run(dec, enc, formula, 1.0, tau)
        _check_draws(logits, fed, u, tau)
        dec._ss_gu = None
        dec.seed_sampling(99, call=2)
        logits, _, fed = _run(dec, enc, formula, 1.0, tau)
        _check_draws(logits, fed, philox.gumbel_uniforms(99, 2, N, T, V), tau)


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_draws_follow_the_softmax_of_the_returned_logits(precision, impl):
    """Pearson statistic of the token counts against the expected counts sum_(b,t) softmax(logits[b][t] / tau) (the draws of one
    row are independent given the logits; a fixed seed: not flaky).  Two calls differ; seed_sampling reproduces a call."""
    from scipy.stats import chisquare
    V, N, T, tau = 12, 64, 40, 1.5
    tfm, p, dec, enc, formula = _setup(V=V, N=N, R=28, T=T, seed=35, precision=precision, impl=impl)
    dec.load_tf_variables({"y_W_o": p["y_W_o"] / 4})             # the glorot scale: logits of about unit spread
    dec.seed_sampling(77, call=0)
    logits, _, first = _run(dec, enc, formula, 1.0, tau)
    _, _, second = _run(dec, enc, formula, 1.0, tau)
    dec.seed_sampling(77, call=0)
    _, _, again = _run(dec, enc, formula, 1.0, tau)
    counts = torch.bincount(first.reshape(-1).cpu(), minlength=V).double().numpy()
    expect = torch.softmax(logits.double() / tau, dim=-1).sum(dim=(0, 1)).cpu().numpy()
    stat, pval = chisquare(counts, expect * counts.sum() / expect.sum())
    print("%s: chi-square %.2f over %d draws, p = %.3f" % (precision, stat, counts.sum(), pval))
    assert pval > 1e-3
    assert (expect / expect.sum()).max() < 0.5                     # not a degenerate distribution
    assert not torch.equal(first, second) and torch.equal(first, again)


# 2 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_coins_of_one_sample_nothing(precision, impl):
    """u = 1: no coin is below p = 1, so fed == formula, the alphas are bit-identical to teacher forcing, and the logits (the
    per-step head instead of the hoisted GEMM) are identical in fp32 — the CUDA-core GEMM sums every output over K in the same
    order at B rows as at T B rows — and within 1e-2 in bf16, where the B-row head runs on mma.sync instead of wgmma."""
    tfm, p, dec, enc, formula = _setup(V=40, N=5, R=28, T=9, seed=37, precision=precision, impl=impl)
    kh, ko = _keeps(*formula.shape, seed=5)
    dec._ss_u = torch.ones(formula.shape).cuda()
    logits, alphas, fed = _run(dec, enc, formula, 1.0, 0.0, kh, ko)
    with torch.no_grad():
        lt, at = dec.train_outputs(enc.cuda(), formula.cuda(), kh, ko)
    assert torch.equal(fed, formula.cuda())
    assert torch.equal(alphas, at)
    err = (logits - lt).abs().max().item()
    print("%s: max |logits - teacher forcing| = %.3e" % (precision, err))
    assert err <= (1e-6 if precision == "fp32" else 1e-2) * max(1.0, lt.abs().max().item())


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_sampled_pass_is_teacher_forcing_on_fed(precision, impl, dropout):
    tfm, p, dec, enc, formula = _setup(V=40, N=4, R=21, T=9, seed=39, precision=precision, impl=impl)
    N, T = formula.shape
    lengths = torch.tensor([9, 6, 3, 7])
    kh, ko = _keeps(N, T, seed=7) if dropout else (None, None)
    runs = []
    for sampled in (True, False):
        x = enc.cuda().requires_grad_(True)
        dec.zero_grad(set_to_none=True)
        if sampled:
            dec.seed_sampling(5)
            logits, alphas = dec.train_outputs(x, formula.cuda(), kh, ko, sampling_prob=1.0, sampling_temperature=0.8)
            fed = dec.last_fed_tokens.clone()
            assert (fed != formula.cuda()).any()
        else:
            logits, alphas = dec.train_outputs(x, fed, kh, ko)
        custom_loss(logits, alphas, formula, lengths).backward()
        runs.append((logits.detach(), alphas.detach(), x.grad.clone(), {k: q.grad.clone() for k, q in dec.named_parameters()}))
    tol = 1e-5 if precision == "fp32" else 1e-2
    for i, what in enumerate(("logits", "alphas", "d enc")):
        assert relerr(runs[0][i], runs[1][i]) < tol, what
    for k in runs[1][3]:
        assert relerr(runs[0][3][k], runs[1][3][k]) < tol, k
    if precision != "fp32":
        return
    # float64 autograd of the oracle on the fed tokens
    pp = {k: v.clone().double().requires_grad_(True) for k, v in p.items()}
    e64 = enc.clone().double().requires_grad_(True)
    lg, al = tfm.decoder_train_logits(pp, e64, fed.cpu(), None if kh is None else kh.double(), None if ko is None else ko.double())
    custom_loss(lg, al, formula, lengths).backward()
    assert relerr(runs[0][0], lg) < 1e-4 and relerr(runs[0][1], al) < 1e-4
    assert relerr(runs[0][2], e64.grad) < 1e-3
    for k, q in runs[0][3].items():
        assert relerr(q, pp[k].grad.reshape(q.shape)) < 1e-3, k


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_p1_without_temperature_is_greedy_decode(precision, impl):
    V, T = 40, 12
    tfm, p, dec, enc, formula = _setup(V=V, N=5, R=28, T=T, seed=41, precision=precision, impl=impl, decoding="greedy")
    _, _, fed = _run(dec, enc, formula, 1.0)
    with torch.no_grad():
        ids = dec.decode(enc.cuda(), max_steps=T).ids
    ref = None
    if precision == "fp32":
        ref = tfm.greedy_decode({k: v.double() for k, v in p.items()}, enc.double(), V - 1, T - 1)
    for b in range(formula.shape[0]):
        g = ids[b].tolist()
        n = g.index(V - 1) + 1 if V - 1 in g else len(g)
        assert fed[b, :n].tolist() == g[:n], b
        if ref is not None:
            r = ref[b].tolist()
            m = r.index(V - 1) + 1 if V - 1 in r else len(r)
            assert fed[b, :min(m, T)].tolist() == r[:min(m, T)], b


# 3 ---------------------------------------------------------------------------------------------------------------------------
def _ref_reward(h, r, end):
    h, r = metrics.truncate_end(h, end), metrics.truncate_end(r, end)
    mx = max(len(h), len(r))
    return np.float32(1.0 if mx == 0 else 1.0 - metrics.levenshtein(h, r) / mx)


def test_tf_reward_and_step_count():
    B, V, end, T = 40, 20, 19, 30
    g = torch.Generator().manual_seed(8)
    hyp, greedy, ref = (torch.randint(0, V - 1, (B, T), generator=g) for _ in range(3))
    for x in (hyp, greedy, ref):
        pos = torch.randint(0, T + 10, (B,), generator=g)
        for b in range(B):
            if pos[b] < T:
                x[b, pos[b]] = end
    hyp[0, 0] = end                             # END at t = 0: n_b = 1
    hyp[1][hyp[1] == end] = 0                   # no END: n_b = T
    hyp[2] = ref[2]                             # an equal pair
    hyp[3] = 1
    ref[3] = 2                                  # a disjoint pair
    r_s, r_g, adv, n = (t.cpu() for t in scst.rewards(hyp.cuda(), ref.cuda(), end, greedy=greedy.cuda(), layout="tf"))
    for b in range(B):
        ws, wg = _ref_reward(hyp[b].tolist(), ref[b].tolist(), end), _ref_reward(greedy[b].tolist(), ref[b].tolist(), end)
        assert r_s[b].item() == ws and r_g[b].item() == wg and adv[b].item() == np.float32(ws - wg), b
        e = [t for t in range(T) if int(hyp[b, t]) == end]
        assert int(n[b]) == min(e[0] + 1, T) if e else int(n[b]) == T, b
    assert int(n[0]) == 1 and int(n[1]) == T and r_s[2] == 1.0 and r_s[3] == 0.0
    # the rewards do not depend on the layout, the step count does
    r_t, _, _, n_t = scst.rewards(hyp.cuda(), ref.cuda(), end, greedy=greedy.cuda())
    assert torch.equal(r_t.cpu(), r_s) and not torch.equal(n_t.cpu(), n)


def test_tf_pg_grad_matches_float64_autograd():
    B, T, V, tau, ldl = 7, 9, 33, 0.7, 64
    g = torch.Generator().manual_seed(4)
    logits = torch.randn(T, B, ldl, generator=g) * 2
    fed = torch.randint(0, V, (B, T), generator=g)
    adv = torch.randn(B, generator=g)
    n_len = torch.tensor([9, 0, 3, 1, 8, 5, 2], dtype=torch.int32)
    dev = "cuda"
    dl = torch.full((B, T, V), 7.0, device=dev)                              # every element must be written
    partial, stats = torch.zeros(B, T, device=dev), torch.zeros(4, device=dev)
    scst.pg_grad_tf(logits.cuda(), fed.cuda(), adv.cuda(), n_len.cuda(), torch.tensor(tau, device=dev), dl, partial, stats)
    x = logits[:, :, :V].double().requires_grad_(True)
    lp = F.log_softmax(x / tau, dim=-1)
    Lw = 0.0
    for b in range(B):
        for t in range(int(n_len[b])):
            Lw = Lw - adv[b].double() * lp[t, b, fed[b, t]]
    Lw = Lw / B
    Lw.backward()
    want = x.grad.transpose(0, 1)
    err = (dl.cpu().double() - want).abs().max().item()
    assert err <= 1e-6 * want.abs().max().item(), err
    assert (dl.cpu()[1] == 0).all()
    assert abs(stats[0].item() - Lw.item()) <= 1e-6 * max(1.0, abs(Lw.item()))
    assert abs(stats[3].item() - n_len.double().mean().item()) < 1e-6


# 4 ---------------------------------------------------------------------------------------------------------------------------
def _scst_loss(logits, fed, adv, n_len, tau):
    N, T, _ = logits.shape
    lp = F.log_softmax(logits / tau, dim=-1).gather(2, fed[:, :, None])[:, :, 0]
    steps = (torch.arange(T, device=lp.device)[None, :] < n_len[:, None].to(lp.device)).to(lp.dtype)
    return -(adv[:, None] * lp * steps).sum() / N


@pytest.mark.parametrize("precision,impl,tol", [("fp32", "simt", 1e-5), ("bf16", "tc", 1e-2)])
def test_fused_step_matches_the_autograd_route(precision, impl, tol):
    V, tau = 30, 0.9
    img, formula, lengths = _tf_batch(V=V, N=3, T=8, seed=24)
    fused, auto = _tf_model(precision, impl, V), _tf_model(precision, impl, V)
    auto.decoder.load_state_dict(fused.decoder.state_dict())
    auto.encoder.load_state_dict(fused.encoder.state_dict())
    u = torch.rand(3, 8, V, generator=torch.Generator().manual_seed(6)).clamp_(1e-6, 1 - 1e-6).cuda()
    fused.decoder._ss_gu = auto.decoder._ss_gu = u                  # the same draws wherever the logits agree
    fused.set_self_critical(tau)
    stats = fused._scst_gradients(img, (formula, lengths), 1.0).clone()
    f = torch.from_numpy(formula).cuda()
    enc = auto.encoder(img)
    with torch.no_grad():
        greedy = auto.decoder.decode(enc.detach(), max_steps=8).ids
    logits, _ = auto.decoder.train_outputs(enc, f, sampling_prob=1.0, sampling_temperature=tau)
    fed = auto.decoder.last_fed_tokens
    assert torch.equal(fed, fused.decoder.last_fed_tokens)
    r_s, r_g, adv, n_len = scst.rewards(fed, f, V - 1, greedy=greedy, layout="tf")
    loss = _scst_loss(logits, fed, adv, n_len, tau)
    loss.backward()
    print("%s: L fused %.6e autograd %.6e; mean r %.4f / %.4f" % (precision, stats[0].item(), loss.item(), stats[1].item(),
                                                                  stats[2].item()))
    assert (adv != 0).any()
    assert abs(stats[0].item() - loss.item()) <= tol * max(abs(loss.item()), 1e-3)
    assert abs(stats[1].item() - r_s.mean().item()) < 1e-6 and abs(stats[2].item() - r_g.mean().item()) < 1e-6
    assert abs(stats[3].item() - n_len.float().mean().item()) < 1e-5
    for mod in ("encoder", "decoder"):
        got = dict(getattr(fused, mod).named_parameters())
        for k, q in getattr(auto, mod).named_parameters():
            assert relerr(got[k].grad, q.grad) < tol, mod + "." + k


def test_a_small_step_along_minus_the_gradient_raises_the_advantage_weighted_log_likelihood():
    V, tau = 40, 1.0
    tfm, p, dec, enc, formula = _setup(V=V, N=6, R=28, T=10, seed=43)
    _, _, fed = _run(dec, enc, formula, 1.0, tau)
    adv = torch.randn(6, generator=torch.Generator().manual_seed(2)).cuda()
    n_len = scst.rewards(fed, formula.cuda(), V - 1, layout="tf")[3]
    x = enc.cuda()

    def objective():
        logits, _ = dec.train_outputs(x, fed)
        return -_scst_loss(logits, fed, adv, n_len, tau) * 6

    dec.zero_grad(set_to_none=True)
    j0 = objective()
    (-j0 / 6).backward()
    with torch.no_grad():
        for q in dec.parameters():
            q.sub_(1e-3 * q.grad)
        j1 = objective()
    print("sum_b adv_b log pi(s_b): %.6f -> %.6f" % (j0.item(), j1.item()))
    assert j1.item() > j0.item()


# 5 ---------------------------------------------------------------------------------------------------------------------------
def test_backward_after_an_intervening_forward_raises():
    tfm, p, dec, enc, formula = _setup(seed=45)
    x = enc.cuda().requires_grad_(True)
    first = dec.train_outputs(x, formula.cuda(), sampling_prob=1.0, sampling_temperature=1.0)
    dec.train_outputs(x, formula.cuda(), sampling_prob=0.5)
    with pytest.raises(_lib.LatexOcrB200Error, match="overwritten"):
        first[0].sum().backward()


@pytest.mark.parametrize("mode", ["sampling", "self_critical"])
def test_one_epoch_then_evaluate(mode):
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    rng = np.random.RandomState(3)
    V = 30
    data = [(rng.randint(0, 256, (32, 64, 1)).astype(np.uint8), list(rng.randint(0, V - 3, 3 + i % 3))) for i in range(6)]
    cfg = _cfg(batch_size=3, n_epochs=1, decoding="greedy", dropout=0.8, lr_init=1e-3, clip=5.0)
    m = Img2SeqModel(cfg, vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc").build_train(cfg)
    before = m.decoder.store.master.clone()
    if mode == "sampling":
        m.set_sampling_prob(0.25)
        score = m._run_train(cfg, data, None, 0, None)
        assert score < 0 and np.isfinite(score) and "perplexity_train" in m.last_epoch_stats
        assert m.decoder.last_fed_tokens.shape[0] == 3
    else:
        m.set_self_critical(1.0)
        score = m._run_train(cfg, data, None, 0, None)
        st = m.last_epoch_stats
        assert score == st["reward_greedy"] and 0.0 <= score <= 1.0
        assert {"scst_loss", "reward_sample", "reward_greedy", "sample_length"} <= set(st)
        assert 1.0 <= st["sample_length"] <= 6.0
        m.set_self_critical(None)
    assert not torch.equal(before, m.decoder.store.master)
    scores = m.evaluate(cfg, data)
    assert np.isfinite(scores["perplexity"]) and "EditDistance" in scores
