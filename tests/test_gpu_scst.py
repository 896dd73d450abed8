"""-m gpu: self-critical sequence training — the Gumbel-max draw inside the time loop (DecoderWithAttention.forward(...,
sampling_temperature=tau)), the edit-distance reward and policy-gradient kernels (latex_ocr_b200.scst), and the fused SCST step
(Img2SeqModel.set_self_critical) against the autograd route, with and without its CUDA graph."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from latex_ocr_b200 import _lib, decode, metrics, philox, scst
from latex_ocr_b200.decoder import DecoderWithAttention
from test_gpu_autograd import _close
from util import build_model

pytestmark = pytest.mark.gpu

PRECISIONS = [("fp32", "simt"), ("bf16", "tc")]


def _oracle():
    from oracle import ref_model as rm
    return rm


def _case(V=50, B=5, R=28, seed=3, lengths=(11, 9, 7, 5, 4)):
    rm = _oracle()
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    formula = torch.randint(0, V, (B, max(lengths)), generator=g)
    enc = torch.randn(B, R, 512, generator=g) * 0.5
    return pe, pd, formula, torch.tensor([[n] for n in lengths[:B]]), enc


def _decoder(pd, V, precision, impl, train):
    dec = DecoderWithAttention(512, 512, 512, V, precision=precision, impl=impl)
    dec.load_state_dict(pd)
    dec.train(train)
    return dec


def _check_draws(preds, fed, u, tau, dl):
    """Every sampled token is argmax(preds / tau + g), g = -log(-log u), in float64 from the returned predictions, wherever the
    top-2 gap exceeds 1e-4; elsewhere it is one of the two."""
    preds = preds.detach().double().cpu()
    u = torch.as_tensor(u).double().cpu()
    fed = fed.cpu()
    exact = near = 0
    for b in range(fed.shape[0]):
        for t in range(1, dl[b]):
            s = preds[b, t - 1] / tau - torch.log(-torch.log(u[b, t]))
            top = torch.topk(s, 2)
            if (top.values[0] - top.values[1]).item() > 1e-4:
                assert int(fed[b, t]) == int(top.indices[0]), (b, t)
                exact += 1
            else:
                assert int(fed[b, t]) in top.indices.tolist(), (b, t)
                near += 1
    assert exact > 0
    return exact, near


# 1 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("R", [28, 868])
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_gumbel_draws_injected_and_philox(precision, impl, R, train):
    V = 60
    pe, pd, formula, lengths, enc = _case(V=V, R=R, seed=5)
    dec = _decoder(pd, V, precision, impl, train=train)
    B, T = formula.shape[0], int(lengths.max()) - 1
    u = torch.rand(B, T, V, generator=torch.Generator().manual_seed(9)).clamp_(1e-6, 1 - 1e-6)
    with torch.no_grad():
        for tau in (0.5, 1.0, 2.0):
            dec._ss_gu = u.cuda()
            preds, caps, dl, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
            _check_draws(preds, dec.last_fed_tokens, u, tau, dl)
            dec._ss_gu = None
            dec.seed_dropout(4242, call=3)
            preds, caps, dl, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
            _check_draws(preds, dec.last_fed_tokens, philox.gumbel_uniforms(4242, 3, B, T, V), tau, dl)
            assert int(dec.dropout_state[1]) == 4


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_draws_follow_the_softmax(precision, impl):
    """fc.weight = 0, fc.bias = fixed logits: every step samples from softmax(bias / tau); the draws of a fixed seed pass a
    chi-square test (fixed seed: not flaky), two calls differ and seed_dropout reproduces them."""
    from scipy.stats import chisquare
    V, B, T, tau = 12, 64, 40, 1.5
    pe, pd, formula, _, enc = _case(V=V, B=B, R=28, seed=21, lengths=(T + 1,) * B)
    lengths = torch.full((B, 1), T + 1)
    bias = torch.linspace(-1.5, 1.0, V)
    pd = dict(pd, **{"fc.weight": torch.zeros_like(pd["fc.weight"]), "fc.bias": bias})
    dec = _decoder(pd, V, precision, impl, train=False)
    dec.seed_dropout(77, call=0)
    with torch.no_grad():
        dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
        first = dec.last_fed_tokens.clone()
        dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
        second = dec.last_fed_tokens.clone()
        dec.seed_dropout(77, call=0)
        dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
        again = dec.last_fed_tokens.clone()
    draws = first[:, 1:].reshape(-1).cpu()
    counts = torch.bincount(draws, minlength=V).double().numpy()
    p = torch.softmax(bias.double() / tau, 0).numpy()
    stat, pval = chisquare(counts, p * counts.sum())
    print("%s: chi-square %.2f over %d draws, p = %.3f" % (precision, stat, counts.sum(), pval))
    assert pval > 1e-3
    assert not torch.equal(first, second) and torch.equal(first, again)


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_without_a_temperature_the_argmax_path_is_unchanged(precision, impl):
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=7)
    dec = _decoder(pd, V, precision, impl, train=True)
    out = []
    with torch.no_grad():
        for kw in ({}, {"sampling_temperature": 0.0}, {"sampling_temperature": None}):
            dec.seed_dropout(31)
            preds, _, _, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=0.5, **kw)
            out.append((preds.clone(), dec.last_fed_tokens.clone()))
    for p_, f_ in out[1:]:
        assert torch.equal(p_, out[0][0]) and torch.equal(f_, out[0][1])


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_sampled_call_equals_teacher_forcing_on_the_samples(precision, impl):
    from test_gpu_autograd import custom_loss
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=13)
    dec = _decoder(pd, V, precision, impl, train=True)
    runs = []
    for sampled in (True, False):
        x = enc.cuda().requires_grad_(True)
        dec.seed_dropout(321)
        if sampled:
            preds, caps, dl, alphas, _ = dec(x, formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=0.8)
            fed = dec.last_fed_tokens.clone()
            assert (fed != caps[:, :fed.shape[1]]).any()
        else:
            f = formula.clone()
            f[:, :fed.shape[1]] = fed.cpu()
            preds, _, dl, alphas, _ = dec(x, f.cuda(), lengths)
        custom_loss(preds, caps, dl, alphas).backward()
        runs.append((preds.detach().clone(), x.grad.clone(), {k: q.grad.clone() for k, q in dec.named_parameters()}))
        dec.zero_grad(set_to_none=True)
    tol = 1e-5 if precision == "fp32" else 1e-2
    print("%s: sampled predictions bit-identical to teacher forcing on the samples: %s" % (precision, torch.equal(*[r[0] for r in runs])))
    _close(runs[0][0], runs[1][0], tol, "predictions")
    _close(runs[0][1], runs[1][1], tol, "d encoder_out", floor=1e-9)
    for k in runs[1][2]:
        if k != "attention.full_att.bias":
            _close(runs[0][2][k], runs[1][2][k], tol, k, floor=1e-9)


# 2 ---------------------------------------------------------------------------------------------------------------------------
def _ref_reward(h, r, end):
    h, r = metrics.truncate_end(h, end), metrics.truncate_end(r, end)
    mx = max(len(h), len(r))
    return np.float32(1.0 if mx == 0 else 1.0 - metrics.levenshtein(h, r) / mx)


@pytest.mark.parametrize("B", [1, 64, 300])
def test_edit_reward_matches_levenshtein(B):
    V, end, L = 20, 19, 152
    g = torch.Generator().manual_seed(B)
    hyp = torch.randint(0, V, (B, L), generator=g)
    greedy = torch.randint(0, V, (B, L - 7), generator=g)
    ref = torch.randint(0, V, (B, L), generator=g)
    # rows with END at random places, some with none
    for x in (hyp, greedy, ref):
        pos = torch.randint(0, x.shape[1] + 20, (B,), generator=g)
        for b in range(B):
            if pos[b] < x.shape[1]:
                x[b, pos[b]] = end
    hyp[0, 0] = end                                         # END at position 0: the empty hypothesis
    if B > 3:
        hyp[1] = ref[1]                                     # equal sequences
        greedy[2] = 0
        ref[2] = 1
        ref[2, 30] = end                                    # disjoint sequences
        ref[3, 0] = end
        hyp[3, 0] = end                                     # both empty
        hyp[4][hyp[4] == end] = 0                           # no END, 152 tokens
        ref[4][ref[4] == end] = 1
    r_s, r_g, adv, n = scst.rewards(hyp.cuda(), ref.cuda(), end, greedy=greedy.cuda())
    r_s, r_g, adv, n = r_s.cpu(), r_g.cpu(), adv.cpu(), n.cpu()
    for b in range(B):
        ws, wg = _ref_reward(hyp[b].tolist(), ref[b].tolist(), end), _ref_reward(greedy[b].tolist(), ref[b].tolist(), end)
        assert r_s[b].item() == ws and r_g[b].item() == wg, b
        assert adv[b].item() == np.float32(ws - wg)
        e = [t for t in range(1, L) if int(hyp[b, t]) == end]
        assert int(n[b]) == (e[0] if e else L - 1)
    assert torch.equal(scst.edit_reward(hyp.cuda(), ref.cuda(), end).cpu(), r_s)
    if B > 3:
        assert r_s[1] == 1.0 and r_s[3] == 1.0 and r_g[2] == 0.0


def test_pg_grad_matches_float64_autograd():
    B, T, V, tau = 7, 9, 33, 0.7
    g = torch.Generator().manual_seed(3)
    ldl = 64
    preds = torch.randn(B, T, ldl, generator=g) * 2
    fed = torch.randint(0, V, (B, T), generator=g)
    adv = torch.randn(B, generator=g)
    n_len = torch.tensor([8, 0, 3, 1, 8, 5, 2], dtype=torch.int32)          # rows end at different steps, one at 0
    dev = "cuda"
    dpred = torch.full((B, T, V), 7.0, device=dev)                            # every element must be written
    partial, stats = torch.zeros(B, T, device=dev), torch.zeros(4, device=dev)
    r_s, r_g = torch.rand(B, generator=g), torch.rand(B, generator=g)
    scst.pg_grad(preds.cuda(), ldl, fed.cuda(), adv.cuda(), n_len.cuda(), torch.tensor(tau, device=dev), B, T, V, dpred, partial,
                 stats, r_sample=r_s.cuda(), r_greedy=r_g.cuda())
    x = preds[:, :, :V].double().requires_grad_(True)
    lp = F.log_softmax(x / tau, dim=-1)
    Lw = 0.0
    for b in range(B):
        for t in range(1, int(n_len[b]) + 1):
            Lw = Lw - adv[b].double() * lp[b, t - 1, fed[b, t]]
    Lw = Lw / B
    Lw.backward()
    _close(dpred, x.grad, 1e-6, "d preds", floor=1e-12)
    assert (dpred.cpu()[1] == 0).all() and (dpred.cpu()[:, T - 1] == 0).all()
    st = stats.cpu().double()
    assert abs(st[0] - Lw.item()) <= 1e-6 * max(1.0, abs(Lw.item()))
    assert abs(st[1] - r_s.double().mean()) < 1e-6 and abs(st[2] - r_g.double().mean()) < 1e-6
    assert abs(st[3] - n_len.double().mean()) < 1e-6


# 3 ---------------------------------------------------------------------------------------------------------------------------
def _scst_loss(preds, fed, adv, n_len, tau):
    B, T, V = preds.shape
    lp = F.log_softmax(preds / tau, dim=-1)
    tok = lp[:, :T - 1].gather(2, fed[:, 1:T].unsqueeze(2)).squeeze(2)                 # log pi(fed[b][t]), t = 1..T-1
    act = (torch.arange(1, T, device=preds.device)[None, :] <= n_len[:, None]).to(preds.dtype)
    return -(adv[:, None] * tok * act).sum() / B


def _autograd_scst_step(m, img, formula, tau, end):
    """The autograd route: greedy rollout under no_grad, sample through dec(...), rewards by scst.rewards, L in plain torch."""
    dec = m.decoder
    N, L = formula.shape
    lens = torch.full((N, 1), L, dtype=torch.long)
    enc = m.encoder(img.cuda())
    with torch.no_grad():
        train = dec.training
        dec.eval()
        dec(enc.detach(), formula.cuda(), lens, sampling_prob=1.0)
        greedy = dec.last_fed_tokens.clone()
        dec.train(train)
    preds, caps, dl, _, _ = dec(enc, formula.cuda(), lens, sampling_prob=1.0, sampling_temperature=tau)
    fed = dec.last_fed_tokens
    r_s, r_g, adv, n_len = scst.rewards(fed, caps, end, greedy=greedy)
    loss = _scst_loss(preds, fed, adv, n_len.long(), tau)
    loss.backward()
    return loss.detach(), fed.clone(), greedy, (r_s, r_g, n_len)


@pytest.mark.parametrize("precision,impl,tol", [("fp32", "simt", 1e-5), ("bf16", "tc", 1e-2)])
def test_fused_step_matches_the_autograd_route(precision, impl, tol):
    rm = _oracle()
    V, tau = 40, 0.9
    pe, pd = rm.init_params(V, seed=41)
    img, formula = rm.synthetic_batch(6, 48, 128, V, 10, 10, seed=42)
    fused = build_model(V, pe, pd, precision, train=True, impl=impl)
    auto = build_model(V, pe, pd, precision, train=True, impl=impl)
    fused.set_self_critical(tau)
    fused.decoder.seed_dropout(77, call=1)
    auto.decoder.seed_dropout(77, call=0)            # the rollout uses up call 0; the sample draws from call 1 in both
    stats = fused.train_step(img.cuda(), formula.cuda(), sync=True).clone()
    loss, fed, greedy, (r_s, r_g, n_len) = _autograd_scst_step(auto, img, formula, tau, V - 1)
    assert torch.equal(fused.decoder.last_fed_tokens, fed)
    assert (fed != greedy).any()
    print("%s: L fused %.6e autograd %.6e; mean r %.4f / %.4f" % (precision, stats[0].item(), loss.item(), stats[1].item(),
                                                                  stats[2].item()))
    assert abs(stats[0].item() - loss.item()) <= tol * max(abs(loss.item()), 1e-3)
    assert abs(stats[1].item() - r_s.mean().item()) < 1e-6 and abs(stats[2].item() - r_g.mean().item()) < 1e-6
    assert abs(stats[3].item() - n_len.float().mean().item()) < 1e-5
    for mod in ("encoder", "decoder"):
        for k, p in getattr(auto, mod).named_parameters():
            q = dict(getattr(fused, mod).named_parameters())[k]
            if k != "attention.full_att.bias":
                _close(q.grad, p.grad, tol, mod + "." + k, floor=1e-9)
    assert torch.equal(auto.decoder.dropout_state.cpu(), fused.decoder.dropout_state.cpu())


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_rollout_is_greedy_decode(precision, impl):
    rm = _oracle()
    V = 40
    pe, pd = rm.init_params(V, seed=51)
    img, formula = rm.synthetic_batch(6, 48, 128, V, 12, 12, seed=52)
    start, end = V - 2, V - 1
    formula[:, 0] = start
    m = build_model(V, pe, pd, precision, train=False, impl=impl)
    m.set_self_critical(1.0)
    m.train_step(img.cuda(), formula.cuda(), sync=True)
    N, L = formula.shape
    T = L - 1
    enc_shape = m.encoder.forward_raw(img.cuda().float(), need_grad=False).shape
    R = enc_shape[1] * enc_shape[2]
    roll = m.decoder._ws[("scst_rollout", N, T, R)]["t"]["fed"].cpu()
    _, si = torch.full((N,), L).sort(dim=0, descending=True)
    m2 = build_model(V, pe, pd, precision, train=False, impl=impl)
    greedy = decode.greedy_decode(m2, img[si], start, end, T)
    assert (roll[:, 0] == start).all()
    for b in range(N):
        g = greedy[b].tolist()[:T - 1]
        e = g.index(end) + 1 if end in g else len(g)
        assert roll[b, 1:1 + e].tolist() == g[:e], b


def _graph_model(V, pe, pd, train):
    m = build_model(V, pe, pd, "bf16", train=train, impl="tc", graph=True)
    for S in m._stores():
        S.refresh_shadow()
    return m


def test_graph_replay_temperature_changes_and_determinism():
    rm = _oracle()
    V = 48
    pe, pd = rm.init_params(V, seed=43)
    img, formula = rm.synthetic_batch(4, 32, 96, V, 8, 8, seed=44)
    N, T = formula.shape[0], formula.shape[1] - 1
    u = torch.rand(N, T, V, generator=torch.Generator().manual_seed(1)).clamp_(1e-6, 1 - 1e-6).cuda()
    first = []
    for graph in (False, True):
        m = _graph_model(V, pe, pd, False) if graph else build_model(V, pe, pd, "bf16", train=False, impl="tc")
        m.decoder._ss_gu = u                            # the same draws in both (the graph's warm-up advances the Philox counter)
        m.set_self_critical(1.0)
        first.append((m.train_step(img, formula, sync=True).clone(), m.decoder.last_fed_tokens.clone()))
    assert torch.equal(first[0][0], first[1][0]) and torch.equal(first[0][1], first[1][1])
    # tau changes between replays without a re-capture: a tiny tau samples the argmax (eval mode: the rollout's tokens, so the
    # two rewards agree), a large one nearly uniform tokens
    m = _graph_model(V, pe, pd, False)
    m.set_self_critical(1e-6)
    st = m.train_step(img, formula, sync=True)
    roll = lambda: next(v for k, v in m.decoder._ws.items() if isinstance(k, tuple) and k[0] == "scst_rollout")["t"]["fed"]
    assert len(m._graphs) == 1 and torch.equal(m.decoder.last_fed_tokens, roll()) and st[1].item() == st[2].item()
    m.set_self_critical(50.0)
    neg = m.getLoss(img, formula)                       # getLoss: -L of the step
    assert len(m._graphs) == 1 and not torch.equal(m.decoder.last_fed_tokens, roll())
    assert neg == -m._graphs[next(iter(m._graphs))]["loss"][0].item()
    m.set_self_critical(None)                           # cross-entropy: its own graph
    m.train_step(img, formula, sync=True)
    assert len(m._graphs) == 2
    # deterministic: two identical steps are bit-identical
    out = []
    with _lib.option(deterministic=1):
        for _ in range(2):
            m = build_model(V, pe, pd, "bf16", train=True, impl="tc")
            m.set_self_critical(0.7)
            m.decoder.seed_dropout(5)
            st = m.train_step(img, formula, sync=True).clone()
            out.append((st, m.decoder.last_fed_tokens.clone(), m.decoder.store.master.clone(), m.encoder.store.master.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_a_small_step_along_minus_the_gradient_raises_the_advantage_weighted_log_likelihood():
    V, tau = 50, 1.0
    pe, pd, formula, _, enc = _case(V=V, B=6, R=28, seed=61, lengths=(12,) * 6)
    lengths = torch.full((6, 1), 12)
    dec = _decoder(pd, V, "fp32", "simt", train=False)
    x = enc.cuda()
    with torch.no_grad():
        dec(x, formula.cuda(), lengths, sampling_prob=1.0, sampling_temperature=tau)
    fed = dec.last_fed_tokens.clone()
    T = fed.shape[1]
    adv = torch.randn(6, generator=torch.Generator().manual_seed(2)).cuda()
    n_len = scst.rewards(fed, formula.cuda(), V - 1)[3].long()
    inp = formula.clone()
    inp[:, :T] = fed.cpu()

    def objective():
        preds, _, _, _, _ = dec(x, inp.cuda(), lengths)
        return -_scst_loss(preds, fed, adv, n_len, tau) * 6          # sum_b adv_b log pi(s_b)

    j0 = objective()
    (-j0 / 6).backward()
    with torch.no_grad():
        for p in dec.parameters():
            if p.grad is not None:
                p.sub_(1e-3 * p.grad)
    with torch.no_grad():
        j1 = objective()
    print("sum_b adv_b log pi(s_b): %.6f -> %.6f" % (j0.item(), j1.item()))
    assert j1.item() > j0.item()
