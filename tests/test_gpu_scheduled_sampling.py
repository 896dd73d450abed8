"""-m gpu: scheduled sampling on the fused decoder (DecoderWithAttention.forward(..., sampling_prob=p), Img2SeqModel.set_sampling_prob):
the token rule on the returned predictions, bit for bit (injected and Philox coins); the sampled call equals teacher forcing on
the tokens it fed (fused path 1e-5 fp32, fp64 oracle 1e-4 outputs / 1e-3 gradients in fp32 and the stated bf16 bounds below);
p = 1 in eval mode feeds what greedy decode emits; u = 1 never samples; the fused train step with and without its CUDA graph;
the bookkeeping rules of the autograd path."""
import pytest
import torch

from latex_ocr_b200 import _lib, philox
from latex_ocr_b200.decoder import DecoderWithAttention
from test_gpu_autograd import _close, custom_loss, reference_get_loss, _optimizers
from util import build_model

pytestmark = pytest.mark.gpu

# bf16 storage + wgmma / mma.sync GEMMs against the fp64 oracle on the same fed tokens, max-abs error over max-abs value (printed
# by the test; the bound leaves room for other seeds, as test_gpu_attention_autograd.py's)
BF16_OUT_BOUND = 3e-2
BF16_GRAD_BOUND = 0.3
PRECISIONS = [("fp32", "simt"), ("bf16", "tc")]


def _oracle():
    from oracle import ref_model as rm
    return rm


def _case(V=50, B=5, R=28, seed=3, lengths=(11, 9, 7, 5, 4)):
    """Rows already sorted by distinct decreasing lengths (the decoder's sort is then the identity)."""
    rm = _oracle()
    pe, pd = rm.init_params(V, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    L = max(lengths)
    formula = torch.randint(0, V, (B, L), generator=g)
    enc = torch.randn(B, R, 512, generator=g) * 0.5
    return pe, pd, formula, torch.tensor([[n] for n in lengths[:B]]), enc


def _decoder(pd, V, precision, impl, train):
    dec = DecoderWithAttention(512, 512, 512, V, precision=precision, impl=impl)
    dec.load_state_dict(pd)
    dec.train(train)
    return dec


def _rule(preds, caps, u, p, decode_lengths):
    """fed[b][t] of the documented rule, from the RETURNED predictions (CPU, torch.argmax: lowest index among equal maxima)."""
    preds, caps, u = preds.detach().float().cpu(), caps.cpu(), u.cpu()
    B, T = u.shape
    fed = caps[:, :T].clone()
    for b in range(B):
        for t in range(1, decode_lengths[b]):
            if u[b, t] < p:
                fed[b, t] = int(torch.argmax(preds[b, t - 1]))
    return fed


# 1 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl", PRECISIONS)
@pytest.mark.parametrize("R", [28, 868])
def test_token_rule_injected_and_philox(precision, impl, R):
    V = 60
    pe, pd, formula, lengths, enc = _case(V=V, R=R, seed=5)
    dec = _decoder(pd, V, precision, impl, train=True)
    B, T = formula.shape[0], int(lengths.max()) - 1
    g = torch.Generator().manual_seed(9)
    u = torch.rand(B, T, generator=g)
    dec._ss_u = u.cuda()
    with torch.no_grad():
        for mask in ("philox", "injected"):
            if mask == "philox":
                preds, caps, dl, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=0.5)
            else:
                # injected dropout multipliers (the parity-test path) through the same entry point the module uses
                enc_s, caps, dl, _ = dec._sorted_inputs(enc.cuda(), formula.cuda(), lengths)
                m = dec.make_dropout_mask(B, T, materialize=True)
                ss = torch.tensor(0.5, device="cuda")
                ws = dec.run_forward(enc_s, caps, dl, with_loss=False, need_grad=False, dropout_mask=m, ss_prob=ss)
                preds = ws["t"]["logits"][:, :, :V]
                dec.last_fed_tokens = ws["t"]["fed"].clone()
            fed = dec.last_fed_tokens.cpu()
            assert torch.equal(fed, _rule(preds, caps, u, 0.5, dl)), mask
            assert (fed != caps[:, :T].cpu()).any()            # something was sampled
    # Philox coins: the host mirror, a new call counter per forward, reproduced by seed_dropout
    dec._ss_u = None
    dec.seed_dropout(4242, call=5)
    runs = []
    with torch.no_grad():
        for call in (5, 6):
            preds, caps, dl, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=0.5)
            uu = torch.from_numpy(philox.sampling_uniforms(4242, call, B, T))
            assert torch.equal(dec.last_fed_tokens.cpu(), _rule(preds, caps, uu, 0.5, dl)), call
            runs.append((preds.clone(), dec.last_fed_tokens.clone()))
        assert int(dec.dropout_state[1]) == 7
        assert not torch.equal(runs[0][1], runs[1][1])
        dec.seed_dropout(4242, call=5)
        preds, _, _, _, _ = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=0.5)
        assert torch.equal(preds, runs[0][0]) and torch.equal(dec.last_fed_tokens, runs[0][1])


# 2 ---------------------------------------------------------------------------------------------------------------------------
def _plain_inputs(formula, fed):
    """Captions whose input tokens are ``fed`` (sorted rows; the targets are taken from the original captions)."""
    f = formula.clone()
    f[:, :fed.shape[1]] = fed.cpu()
    return f


def _sampled_and_plain(dec, formula, lengths, enc, p, seed):
    x = enc.cuda().requires_grad_(True)
    dec.seed_dropout(seed)
    preds, caps, dl, alphas, _ = dec(x, formula.cuda(), lengths, sampling_prob=p)
    custom_loss(preds, caps, dl, alphas).backward()
    fed = dec.last_fed_tokens.clone()
    got = (preds.detach().clone(), alphas.detach().clone(), x.grad.clone(),
           {k: q.grad.detach().clone() for k, q in dec.named_parameters()}, dec._ws_for(*_shape(dec, formula, lengths, enc))["t"]["hall"].clone())
    dec.zero_grad(set_to_none=True)
    y = enc.cuda().requires_grad_(True)
    dec.seed_dropout(seed)                       # same dropout masks: the sampled call consumed exactly this call counter
    preds2, _, dl2, alphas2, _ = dec(y, _plain_inputs(formula, fed).cuda(), lengths)
    custom_loss(preds2, caps, dl2, alphas2).backward()       # targets: the original captions
    want = (preds2.detach().clone(), alphas2.detach().clone(), y.grad.clone(),
            {k: q.grad.detach().clone() for k, q in dec.named_parameters()}, dec._ws_for(*_shape(dec, formula, lengths, enc))["t"]["hall"].clone())
    dec.zero_grad(set_to_none=True)
    return fed, caps, dl, got, want


def _shape(dec, formula, lengths, enc):
    return enc.shape[0], int(lengths.max()) - 1, enc.shape[1]


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_sampled_call_equals_teacher_forcing_on_fed_tokens(precision, impl):
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=7)
    dec = _decoder(pd, V, precision, impl, train=True)
    fed, caps, dl, got, want = _sampled_and_plain(dec, formula, lengths, enc, 0.5, 321)
    assert (fed != caps[:, :fed.shape[1]]).any()
    tol = 1e-5 if precision == "fp32" else 1e-2          # bf16: the predictions feed bf16 d logits / d gates mirrors
    print("%s: sampled predictions bit-identical to the teacher-forced call on fed: %s" % (precision, torch.equal(got[0], want[0])))
    _close(got[0], want[0], tol, "predictions")
    _close(got[1], want[1], tol, "alphas")
    _close(got[2], want[2], tol, "d encoder_out", floor=1e-9)
    for k in want[3]:
        if k != "attention.full_att.bias":
            _close(got[3][k], want[3][k], tol, k, floor=1e-9)


@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_sampled_call_vs_float64_oracle(precision, impl):
    rm = _oracle()
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=11)
    dec = _decoder(pd, V, precision, impl, train=False)
    x = enc.cuda().requires_grad_(True)
    preds, caps, dl, alphas, _ = dec(x, formula.cuda(), lengths, sampling_prob=0.6)
    custom_loss(preds, caps, dl, alphas).backward()
    fed = dec.last_fed_tokens.cpu()
    assert (fed != caps[:, :fed.shape[1]].cpu()).any()
    if precision == "bf16":         # the oracle sees what the kernels see: bf16-rounded weights and inputs
        pdd = {k: (v.bfloat16().double() if v.dim() == 2 and "full_att" not in k else v.double()).requires_grad_(True)
               for k, v in pd.items()}
        xd = enc.bfloat16().double().requires_grad_(True)
    else:
        pdd = {k: v.double().requires_grad_(True) for k, v in pd.items()}
        xd = enc.double().requires_grad_(True)
    p2, c2, dl2, a2, _ = rm.decoder_forward(pdd, xd, _plain_inputs(formula, fed), lengths)
    assert dl2 == dl
    custom_loss(p2, caps.cpu(), dl2, a2).backward()

    def err(g, w):
        g, w = g.detach().double().cpu().reshape(-1), w.detach().double().cpu().reshape(-1)
        assert torch.isfinite(g).all()
        return (g - w).abs().max().item() / (w.abs().max().item() + 1e-30)
    out = max(err(preds, p2), err(alphas, a2))
    grads = {"d encoder_out": err(x.grad, xd.grad)}
    for k, q in dec.named_parameters():
        if k != "attention.full_att.bias":
            grads[k] = err(q.grad, pdd[k].grad)
    print("%s vs fp64 oracle on the fed tokens: outputs %.3e, gradients max %.3e" % (precision, out, max(grads.values())))
    ob, gb = (1e-4, 1e-3) if precision == "fp32" else (BF16_OUT_BOUND, BF16_GRAD_BOUND)
    assert out < ob
    for k, e in grads.items():
        assert e < gb, (k, e)


# 3 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_p1_eval_feeds_the_greedy_tokens(precision, impl):
    """p = 1 in eval mode: step t feeds the argmax of step t-1, exactly what lo_decoder_greedy emits when it starts from the same
    first token.  Full-length rows: greedy runs every row at every step, and so does the sampled call (with shorter rows the
    attention kernels would split fewer rows differently and the sums would round differently)."""
    import ctypes
    V, B, T = 60, 8, 12
    pe, pd, formula, _, enc = _case(V=V, B=B, R=35, seed=13, lengths=(T + 1,) * B)
    lengths = torch.full((B, 1), T + 1)
    start = V - 2
    formula[:, 0] = start
    dec = _decoder(pd, V, precision, impl, train=False)
    with torch.no_grad():
        _, _, _, _, sort_ind = dec(enc.cuda(), formula.cuda(), lengths, sampling_prob=1.0)
        fed = dec.last_fed_tokens.clone()
        enc_s = enc.cuda()[sort_ind].to(dec.tdtype).contiguous()       # greedy on the same rows in the same order
        ws = dec.workspace(B, T, enc.shape[1], need_grad=False)
        for t in range(T):
            ws["bt"][t] = B
        a = dec.fill_args(ws, enc_s, B, T, enc.shape[1], has_dropout=False)
        tokens = torch.zeros(B, T, dtype=torch.int64, device="cuda")
        finished = torch.zeros(B, dtype=torch.int32, device="cuda")
        _lib.check(_lib.lib().lo_decoder_greedy(ctypes.byref(a), start, V - 1, T, tokens.data_ptr(), finished.data_ptr(),
                                                _lib.stream_ptr()))
    assert (fed[:, 0] == start).all()
    assert torch.equal(fed[:, 1:], tokens[:, :T - 1])


# 4 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl", PRECISIONS)
def test_never_sampling_through_the_sampling_path(precision, impl):
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=17)
    dec = _decoder(pd, V, precision, impl, train=True)
    B, T = formula.shape[0], int(lengths.max()) - 1
    dec._ss_u = torch.ones(B, T, device="cuda")
    fed, caps, dl, got, want = _sampled_and_plain(dec, formula, lengths, enc, 0.5, 99)
    assert torch.equal(fed, caps[:, :T])
    assert torch.equal(got[4], want[4])                  # hidden states: the same cell on the same tokens
    assert torch.equal(got[1], want[1])                  # alphas
    tol = 1e-5 if precision == "fp32" else 1e-2
    _close(got[0], want[0], tol, "predictions")
    _close(got[2], want[2], tol, "d encoder_out", floor=1e-9)
    for k in want[3]:
        if k != "attention.full_att.bias":
            _close(got[3][k], want[3][k], tol, k, floor=1e-9)


# 5 ---------------------------------------------------------------------------------------------------------------------------
def _get_loss_sampled(model, p, img, formula):
    """reference_get_loss with the decoder call given sampling_prob = p."""
    import torch.nn as nn
    eo, do = _optimizers(model)
    orig = model.decoder.forward
    model.decoder.forward = lambda *a: orig(*a, sampling_prob=p)
    try:
        return reference_get_loss(model, eo, do, nn.CrossEntropyLoss(), img, formula)
    finally:
        del model.decoder.forward


@pytest.mark.parametrize("precision,impl,tol", [("fp32", "simt", 1e-5), ("bf16", "tc", 1e-2)])
def test_fused_step_matches_autograd_step(precision, impl, tol):
    rm = _oracle()
    V = 64
    pe, pd = rm.init_params(V, seed=41)
    img, formula = rm.synthetic_batch(6, 48, 128, V, 10, 10, seed=42)
    fused = build_model(V, pe, pd, precision, train=True, impl=impl)
    auto = build_model(V, pe, pd, precision, train=True, impl=impl)
    fused.set_sampling_prob(0.25)
    fused.decoder.seed_dropout(77)
    auto.decoder.seed_dropout(77)
    loss = fused.train_step(img.cuda(), formula.cuda(), sync=True)
    neg = _get_loss_sampled(auto, 0.25, img, formula)
    assert torch.equal(fused.decoder.last_fed_tokens, auto.decoder.last_fed_tokens)
    assert (auto.decoder.last_fed_tokens != formula[:, :-1].cuda()).any()
    assert abs(-neg - loss[0].item()) / loss[0].item() < tol
    for mod in ("encoder", "decoder"):
        for k, p in getattr(auto, mod).named_parameters():
            q = dict(getattr(fused, mod).named_parameters())[k]
            if k != "attention.full_att.bias":
                _close(p.grad, q.grad, tol, mod + "." + k, floor=1e-9)
    assert torch.equal(auto.decoder.dropout_state.cpu(), fused.decoder.dropout_state.cpu())


def _graph_model(V, pe, pd):
    """A graphed bf16 model whose shadows are cast before its first step: the first graph step snapshots the stores (bf16 shadows
    included) before its warm-up and restores that snapshot, so an uncast shadow would make it train on other weights than the
    eager arm."""
    m = build_model(V, pe, pd, "bf16", train=False, impl="tc", graph=True)
    for S in m._stores():
        S.refresh_shadow()
    return m


def test_fused_step_graph_replay_and_p_changes():
    rm = _oracle()
    V = 48
    pe, pd = rm.init_params(V, seed=43)
    img, formula = rm.synthetic_batch(4, 32, 96, V, 8, 8, seed=44)
    B, T = formula.shape[0], formula.shape[1] - 1
    u = torch.rand(B, T, generator=torch.Generator().manual_seed(1)).cuda()
    losses, feds = [], []
    for graph in (False, True):
        m = _graph_model(V, pe, pd) if graph else build_model(V, pe, pd, "bf16", train=False, impl="tc")
        m.decoder._ss_u = u                        # the same coins in both (the graph's warm-up steps advance the Philox counter)
        m.set_sampling_prob(0.5)
        losses.append([m.train_step(img, formula, sync=True)[0].item()])
        feds.append(m.decoder.last_fed_tokens.clone())
        losses[-1] += [m.train_step(img, formula, sync=True)[0].item() for _ in range(2)]
    assert torch.equal(feds[0], feds[1]) and losses[0][0] == losses[1][0]     # the first step: the same launches on the same data
    # later steps: fp32 atomics differ at rounding level between runs, which Adam amplifies (test_gpu_parity.py) and an argmax
    # between near-equal logits can turn into another fed token
    for a, b in zip(*losses):
        assert abs(a - b) / abs(a) < 1e-2, losses
    # p changes between replays without a re-capture: constant coins 0.5, so p = 0.25 never samples and p = 0.75 always does
    u2 = torch.full((B, T), 0.5, device="cuda")
    m2 = _graph_model(V, pe, pd)
    m2.decoder._ss_u = u2
    m2.set_sampling_prob(0.25)
    m2.train_step(img, formula, sync=True)
    _, si = torch.full((B,), T + 1).sort(dim=0, descending=True)          # the train step's row order (all rows equally long)
    caps = formula[si][:, :T].cuda()
    assert len(m2._graphs) == 1 and torch.equal(m2.decoder.last_fed_tokens, caps)
    m2.set_sampling_prob(0.75)
    m2.train_step(img, formula, sync=True)
    assert len(m2._graphs) == 1 and not torch.equal(m2.decoder.last_fed_tokens, caps)
    m2._ss_prob_dev.fill_(0.0)                     # p = 0 inside the sampling graph: the teacher tokens
    m2.train_step(img, formula, sync=True)
    assert len(m2._graphs) == 1 and torch.equal(m2.decoder.last_fed_tokens, caps)
    m2.set_sampling_prob(0.0)                      # the teacher-forced step: its own graph, no fed record
    m2.train_step(img, formula, sync=True)
    assert len(m2._graphs) == 2 and m2.decoder.last_fed_tokens is None


def test_fused_step_deterministic_is_bit_identical():
    rm = _oracle()
    V = 48
    pe, pd = rm.init_params(V, seed=45)
    img, formula = rm.synthetic_batch(4, 32, 96, V, 8, 8, seed=46)
    out = []
    with _lib.option(deterministic=1):
        for _ in range(2):
            m = build_model(V, pe, pd, "bf16", train=True, impl="tc")
            m.set_sampling_prob(0.25)
            m.decoder.seed_dropout(5)
            loss = m.train_step(img, formula, sync=True).clone()
            out.append((loss, m.decoder.last_fed_tokens.clone(), m.decoder.store.master.clone(), m.encoder.store.master.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


# 6 ---------------------------------------------------------------------------------------------------------------------------
def test_bookkeeping_of_the_sampled_autograd_path():
    V = 50
    pe, pd, formula, lengths, enc = _case(V=V, seed=19)
    dec = _decoder(pd, V, "fp32", "simt", train=True)
    B, T = formula.shape[0], int(lengths.max()) - 1
    dec._ss_u = torch.rand(B, T, generator=torch.Generator().manual_seed(2)).cuda()

    def step():
        x = enc.cuda().requires_grad_(True)
        dec.seed_dropout(8)
        preds, caps, dl, alphas, _ = dec(x, formula.cuda(), lengths, sampling_prob=0.5)
        custom_loss(preds, caps, dl, alphas).backward()

    step()
    once = {k: q.grad.clone() for k, q in dec.named_parameters()}
    step()                                                 # no zero_grad: accumulates
    for k, q in dec.named_parameters():
        _close(q.grad, 2 * once[k], 1e-5, k, floor=1e-9)
    dec.zero_grad(set_to_none=True)
    dec.fine_tune_embeddings(False)                        # frozen: no gradient
    step()
    assert dec.embedding.weight.grad is None and dec.fc.weight.grad is not None
    dec.fine_tune_embeddings(True)
    # an interleaved forward of the same shape overwrites the saved state (fed included): the first backward refuses
    x = enc.cuda().requires_grad_(True)
    first = dec(x, formula.cuda(), lengths, sampling_prob=0.5)
    dec(x, formula.cuda(), lengths, sampling_prob=0.5)
    with pytest.raises(_lib.LatexOcrB200Error):
        first[0].sum().backward()
