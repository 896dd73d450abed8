"""-m gpu: training the row-encoder extension (BASELINE.json configs[3], latex_ocr_b200/ext.py) through loss.backward() —
autograd of RowEncoder.forward and of the two-layer decoder TwoLayerDecoder (Img2SeqRowModel.decoder2) on the CUDA kernels,
against the fp64 CPU definition oracle/ref_ext.py with autograd, the fused Img2SeqRowModel step, and the bookkeeping rules of torch
(gradient accumulation, frozen parameters, optimizer visibility, stale saved state, dropout replay).  Tolerances: fp32 — oracle
1e-4 of max-abs on outputs and 1e-3 on gradients (as test_gpu_ext.py), fused step 1e-5; bf16 + wgmma — the stated bound
BF16_TOL / BF16_TOL_PARAM of max-abs against the fp32-parameter oracle, and 1e-2 against the fused bf16 step."""
import pytest
import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import pack_padded_sequence

from latex_ocr_b200 import _lib
from latex_ocr_b200.params import grad_view
from util import Cfg

pytestmark = pytest.mark.gpu

V = 50
# stated bounds: the whole chain in bf16 storage (six convs, the biLSTM, both decoder layers; fp32 accumulation) against fp64 with
# the fp32 parameters.  Measured on an H100 over the eight cases: outputs and d feat / d encoder_out at most 9e-3 of max-abs,
# parameter gradients at most 0.17 (decoder_att.weight, then cnn.0 at 0.13) — the kernels' bf16 error: the autograd gradients
# are within 2e-3 of the fused bf16 step's
BF16_TOL = 2e-2
BF16_TOL_PARAM = 0.25
MODS = ("encoder", "row_encoder", "decoder", "layer2")


def _oracles():
    from oracle import ref_ext as rx
    from oracle import ref_model as rm
    return rm, rx


def _model(pe, prow, pd, p2, precision="fp32", train=False):
    from latex_ocr_b200.ext import Img2SeqRowModel
    m = Img2SeqRowModel(Cfg(), n_tok=V, device="cuda", precision=precision, impl="tc" if precision == "bf16" else "simt")
    m.build_train()
    for mod, sd in zip(MODS, (pe, prow, pd, p2)):
        getattr(m, mod).load_state_dict(sd)
    m.train_mode(train)
    return m


def _case(seed=3, B=4):
    """Parameters, a batch of 32x64 images (feature map 2x6, R = 12) and ragged caption lengths (all distinct)."""
    rm, rx = _oracles()
    pe, pd = rm.init_params(V, seed=seed)
    prow, p2 = rx.init_params_ext(seed=seed + 1)
    img, formula = rm.synthetic_batch(B, 32, 64, V, 3, 9, seed=seed + 2)
    L = formula.shape[1]
    lengths = torch.tensor([[L - 5], [L], [L - 2], [L - 3]])[:B]
    return pe, prow, pd, p2, img, formula, lengths


def _params(m):
    return [(mod + "." + k, p) for mod in MODS for k, p in getattr(m, mod).named_parameters()]


def custom_loss(preds, caps, decode_lengths, alphas):
    """Label-smoothed CE over the decoded positions + a regulariser whose weight changes with t (so d loss / d alpha does)."""
    B, T, _ = preds.shape
    dev = preds.device
    act = (torch.arange(T, device=dev)[None, :] < torch.tensor(decode_lengths, device=dev)[:, None]).to(preds.dtype)
    lp = F.log_softmax(preds, dim=-1)
    nll = -lp.gather(2, caps[:, 1:T + 1].unsqueeze(2)).squeeze(2)
    ce = ((0.9 * nll - 0.1 * lp.mean(dim=2)) * act).sum() / act.sum()
    w = torch.linspace(0.5, 1.5, T, dtype=preds.dtype, device=dev)
    return ce + 0.7 * ((1. - (alphas * w[None, :, None]).sum(dim=1)) ** 2).mean()


def reference_loss(preds, caps, decode_lengths, alphas):
    """img2seq_torch.py:147-159: CE over the packed positions + the doubly-stochastic regulariser."""
    scores = pack_padded_sequence(preds, decode_lengths, batch_first=True).data
    targets = pack_padded_sequence(caps[:, 1:], decode_lengths, batch_first=True).data
    return F.cross_entropy(scores, targets) + ((1. - alphas.sum(dim=1)) ** 2).mean()


def _err(got, want):
    """max-abs error over max-abs of the reference."""
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    assert torch.isfinite(got).all()
    return (got - want).abs().max().item() / max(want.abs().max().item(), 1e-30)


def _close(got, want, tol, name, floor=2e-8):
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    assert torch.isfinite(got).all(), name
    err = (got - want).abs().max().item()
    assert err <= tol * want.abs().max().item() + floor, (name, err, want.abs().max().item())


def _oracle_chain(pe, prow, pd, p2, img, formula, lengths, mask):
    """fp64 autograd of encoder -> row encoder -> two-layer decoder (ragged: outputs at t >= len_b zeroed, as
    DecoderWithAttention does) -> custom_loss.  ``mask``: dropout multipliers [B,T,D] in sorted row order, or None."""
    rm, rx = _oracles()
    P = [{k: v.double().requires_grad_(True) for k, v in d.items()} for d in (pe, prow, pd, p2)]
    feat = rm.encoder_forward(P[0], img.double())
    feat.retain_grad()
    enc = rx.row_encoder_forward(P[1], feat)
    enc.retain_grad()
    N = enc.shape[0]
    lens, si = lengths.squeeze(1).sort(dim=0, descending=True)
    dl = (lens - 1).tolist()
    T = max(dl)
    caps = formula[si]
    preds, alphas = rx.decoder2_forward(P[2], P[3], enc.reshape(N, -1, enc.shape[3])[si], caps, T,
                                        None if mask is None else mask.double())
    act = (torch.arange(T)[None, :] < torch.tensor(dl)[:, None]).double()[:, :, None]
    preds, alphas = preds * act, alphas * act
    custom_loss(preds, caps, dl, alphas).backward()
    grads = {mod + "." + k: v.grad for mod, d in zip(MODS, P) for k, v in d.items()}
    return preds.detach(), alphas.detach(), feat.grad, enc.grad, grads


# 1 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("layout", ["NHWC", "NRC"])
def test_custom_loss_vs_fp64_oracle(precision, dropout, layout):
    pe, prow, pd, p2, img, formula, lengths = _case()
    B = img.shape[0]
    T = int(lengths.max()) - 1
    mask = (torch.rand(B, T, 512, generator=torch.Generator().manual_seed(5)) >= 0.5).float() * 2.0 if dropout else None
    want_p, want_a, want_dfeat, want_denc, want_g = _oracle_chain(pe, prow, pd, p2, img, formula, lengths, mask)
    m = _model(pe, prow, pd, p2, precision)
    if mask is not None:            # injected multipliers in place of the in-kernel draw (sorted row order, like the oracle's)
        m.decoder.make_dropout_mask = lambda B_, T_, materialize=False: mask.cuda()
    feat = m.encoder(img.cuda())
    feat.retain_grad()
    enc = m.row_encoder(feat)
    enc.retain_grad()
    x = enc if layout == "NHWC" else enc.view(B, -1, enc.shape[3])
    preds, caps, dl, alphas, _ = m.decoder2(x, formula.cuda(), lengths)
    assert preds.shape == (B, T, V) and alphas.shape == (B, T, 12) and dl == sorted(dl, reverse=True)
    custom_loss(preds, caps, dl, alphas).backward()
    assert feat.grad.shape == feat.shape and enc.grad.shape == enc.shape
    errs = {"predictions": _err(preds, want_p), "alphas": _err(alphas, want_a), "d feat": _err(feat.grad, want_dfeat),
            "d encoder_out": _err(enc.grad, want_denc)}
    for k, p in _params(m):
        if k != "decoder.attention.full_att.bias":      # exactly 0 (softmax shift invariance): rounding noise on both sides
            assert p.grad is not None, k
            errs[k] = _err(p.grad, want_g[k])
    print("\n[%s dropout=%s %s] outputs: %s; worst: %s" % (precision, dropout, layout, [(k, errs[k]) for k in list(errs)[:4]],
                                                          sorted(errs.items(), key=lambda kv: -kv[1])[:3]))
    for k, e in errs.items():
        if precision == "bf16":
            tol = BF16_TOL if k in ("predictions", "alphas", "d feat", "d encoder_out") else BF16_TOL_PARAM
        else:
            tol = 1e-4 if k in ("predictions", "alphas") else 1e-3
        assert e < tol, (k, e)


# 2 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 1e-2)])
def test_reference_loss_through_autograd_matches_fused_step(precision, tol):
    """Every row at the padded length, in-kernel Philox dropout from the same {seed, call}: the gradients of the reference loss
    through autograd are those of the fused step (fp32: 1e-5 of max-abs; bf16: 1e-2, d logits reach the bf16 mirror of the fc
    backward through another rounding)."""
    pe, prow, pd, p2, img, formula, _ = _case(seed=11)
    B, L = formula.shape
    fused = _model(pe, prow, pd, p2, precision, train=True)
    auto = _model(pe, prow, pd, p2, precision, train=True)
    fused.decoder.seed_dropout(77, call=2)
    auto.decoder.seed_dropout(77, call=2)
    loss = fused.train_step(img.cuda(), formula.cuda(), sync=True)
    preds, caps, dl, alphas, _ = auto.decoder2(auto.row_encoder(auto.encoder(img.cuda())), formula.cuda(),
                                               torch.full((B, 1), L, dtype=torch.long))
    ref = reference_loss(preds, caps, dl, alphas)
    ref.backward()
    assert abs(ref.item() - loss[0].item()) <= 1e-5 * abs(loss[0].item())
    want = dict(_params(fused))
    errs = {}
    for k, p in _params(auto):
        if k != "decoder.attention.full_att.bias":
            errs[k] = _err(p.grad, want[k].grad)
            _close(p.grad, want[k].grad, tol, k, floor=1e-9)
    print("\n[%s] worst: %s" % (precision, sorted(errs.items(), key=lambda kv: -kv[1])[:3]))
    assert torch.equal(auto.decoder.dropout_state.cpu(), fused.decoder.dropout_state.cpu())     # one Philox call either way


# 3 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_grad_enabled_outputs_equal_no_grad_outputs(precision):
    pe, prow, pd, p2, img, formula, lengths = _case(seed=21)
    m = _model(pe, prow, pd, p2, precision, train=True)
    outs = []
    for grad in (False, True):
        m.decoder.seed_dropout(5)
        with torch.set_grad_enabled(grad):
            feat = m.encoder(img.cuda())
            y = m.row_encoder(feat)
            y_saved = y.detach().clone()              # the no_grad fp32 output is the cached buffer: copy it before reuse
            res = m.decoder2(y, formula.cuda(), lengths)
        assert (y.grad_fn is not None) == grad and (res[0].grad_fn is not None) == grad and (res[3].grad_fn is not None) == grad
        outs.append((y_saved, res[0].detach().clone(), res[1], res[2], res[3].detach().clone(), res[4]))
    for a, b in zip(*outs):
        assert a == b if isinstance(a, list) else torch.equal(a, b)


# 4 ---------------------------------------------------------------------------------------------------------------------------
def test_gradient_bookkeeping():
    pe, prow, pd, p2, img, formula, lengths = _case(seed=31)
    m = _model(pe, prow, pd, p2, "fp32")
    params = _params(m)

    def step():
        preds, caps, dl, alphas, _ = m.decoder2(m.row_encoder(m.encoder(img.cuda())), formula.cuda(), lengths)
        custom_loss(preds, caps, dl, alphas).backward()

    def zero_grad(set_to_none):
        for mod in MODS:
            getattr(m, mod).zero_grad(set_to_none=set_to_none)

    step()
    once = {k: p.grad.clone() for k, p in params}
    step()                                                   # no zero_grad: accumulates
    for k, p in params:
        _close(p.grad, 2 * once[k], 1e-5, k, floor=1e-9)
    for set_to_none in (True, False):
        zero_grad(set_to_none)
        for k, p in params:
            assert (p.grad is None) if set_to_none else (p.grad.abs().max().item() == 0), k
        step()
        for k, p in params:
            _close(p.grad, once[k], 1e-5, k, floor=1e-9)
    # frozen parameters get no gradient
    frozen = (m.row_encoder.lstm.weight_ih_l0_reverse, m.layer2.cell.bias_hh, m.decoder.embedding.weight)
    for p in frozen:
        p.requires_grad_(False)
    zero_grad(True)
    step()
    for k, p in params:
        assert (p.grad is None) == (not p.requires_grad), k
    assert all(p.grad is None for p in frozen)
    # a fused step afterwards leaves its gradients in p.grad, which alias the flat buffers again
    for p in frozen:
        p.requires_grad_(True)
    m.getLoss(img, formula)
    for mod in MODS:
        M = getattr(m, mod)
        for k, p in M.named_parameters():
            gv = grad_view(M.store, p)
            assert p.grad is not None and p.grad.data_ptr() == gv.data_ptr() and torch.equal(p.grad, gv), (mod, k)
        assert M.store.grad.abs().sum().item() > 0, mod


# 5 ---------------------------------------------------------------------------------------------------------------------------
def test_torch_optimizer_step_is_visible_to_the_next_forward():
    pe, prow, pd, p2, img, formula, lengths = _case(seed=41)
    m = _model(pe, prow, pd, p2, "bf16")
    opt = torch.optim.Adam(list(m.row_encoder.parameters()) + list(m.layer2.parameters()), lr=1e-2)
    preds, caps, dl, alphas, _ = m.decoder2(m.row_encoder(m.encoder(img.cuda())), formula.cuda(), lengths)
    custom_loss(preds, caps, dl, alphas).backward()
    opt.step()
    sds = [{k: v.detach().cpu().clone() for k, v in getattr(m, mod).state_dict().items()} for mod in MODS]
    assert not torch.equal(sds[1]["lstm.weight_hh_l0"], prow["lstm.weight_hh_l0"])
    assert not torch.equal(sds[3]["cell.weight_ih"], p2["cell.weight_ih"])
    fresh = _model(*sds, precision="bf16")
    outs = []
    with torch.no_grad():
        for mm in (m, fresh):
            y = mm.row_encoder(mm.encoder(img.cuda())).clone()
            res = mm.decoder2(y, formula.cuda(), lengths)
            outs.append((y, res[0], res[3]))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# 6 ---------------------------------------------------------------------------------------------------------------------------
def test_backward_of_overwritten_forward_state_raises():
    pe, prow, pd, p2, img, formula, lengths = _case(seed=51)
    m = _model(pe, prow, pd, p2, "fp32")
    g = torch.Generator().manual_seed(52)
    # row encoder: a later forward of the same shape, and one of another shape that shares the per-direction state
    feat = (torch.randn(2, 2, 6, 512, generator=g) * 0.5).cuda().requires_grad_(True)
    for other in (feat, (torch.randn(4, 1, 6, 512, generator=g) * 0.5).cuda()):
        y = m.row_encoder(feat)
        m.row_encoder(other)
        with pytest.raises(_lib.LatexOcrB200Error):
            y.sum().backward()
    enc = (torch.randn(4, 12, 512, generator=g) * 0.5).cuda().requires_grad_(True)
    f, l_ = formula.cuda(), lengths
    # two-layer decoder: the same shape again; another R with the same (B, T), which rewrites layer 2's state only; the plain
    # DecoderWithAttention of the same shape, which rewrites layer 1's
    for later in (lambda: m.decoder2(enc, f, l_), lambda: m.decoder2(enc[:, :8], f, l_), lambda: m.decoder(enc, f, l_)):
        first = m.decoder2(enc, f, l_)
        later()
        with pytest.raises(_lib.LatexOcrB200Error):
            first[0].sum().backward()
    first = m.decoder2(enc, f, l_)                            # and nothing raises without a later forward
    first[0].sum().backward()
    assert enc.grad is not None and enc.grad.abs().sum().item() > 0


# 7 ---------------------------------------------------------------------------------------------------------------------------
def test_dropout_replay_with_interleaved_forward():
    pe, prow, pd, p2, img, formula, lengths = _case(seed=61)
    m = _model(pe, prow, pd, p2, "fp32", train=True)
    enc = (torch.randn(4, 2, 6, 512, generator=torch.Generator().manual_seed(62)) * 0.5).cuda()
    dec2 = m.decoder2

    def grads():
        return {k: p.grad.clone() for k, p in dec2.named_parameters()}

    m.decoder.seed_dropout(99, call=3)
    x = enc.clone().requires_grad_(True)
    preds, caps, dl, alphas, _ = dec2(x, formula.cuda(), lengths)
    custom_loss(preds, caps, dl, alphas).backward()
    want_dx, want = x.grad.clone(), grads()
    dec2.zero_grad(set_to_none=True)
    m.decoder.seed_dropout(99, call=3)
    x = enc.clone().requires_grad_(True)
    preds, caps, dl, alphas, _ = dec2(x, formula.cuda(), lengths)
    other = dec2(enc[:3, :1], formula[:3, :6].cuda(), torch.tensor([[6], [5], [4]]))     # another shape, another mask
    other[0].sum().backward()
    dec2.zero_grad(set_to_none=True)
    custom_loss(preds, caps, dl, alphas).backward()
    _close(x.grad, want_dx, 1e-5, "d encoder_out", floor=1e-9)
    got = grads()
    for k in want:
        _close(got[k], want[k], 1e-5, k, floor=1e-9)


# 8 ---------------------------------------------------------------------------------------------------------------------------
def test_twelve_bf16_adam_steps_through_autograd_lower_the_loss():
    pe, prow, pd, p2, img, formula, _ = _case(seed=71)
    B, L = formula.shape
    m = _model(pe, prow, pd, p2, "bf16", train=True)
    opt = torch.optim.Adam([p for mod in MODS for p in getattr(m, mod).parameters()], lr=1e-3)
    lengths = torch.full((B, 1), L, dtype=torch.long)
    losses = []
    for _ in range(13):
        preds, caps, dl, alphas, _ = m.decoder2(m.row_encoder(m.encoder(img.cuda())), formula.cuda(), lengths)
        loss = reference_loss(preds, caps, dl, alphas)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(map(lambda v: v == v, losses)) and losses[-1] < losses[0], losses
