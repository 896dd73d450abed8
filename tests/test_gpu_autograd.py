"""-m gpu: training through loss.backward() — autograd of EncoderCNN.forward and DecoderWithAttention.forward on the CUDA
kernels (lo_decoder_backward in its generic mode, EncoderCNN.backward_raw), against the golden fixtures of the reference,
the fused train step, the CPU oracle and the bookkeeping rules of torch (gradient accumulation, frozen parameters, optimizer
visibility, stale saved state).  Tolerances: fp32 — golden 1e-3 of each gradient's max-abs (as test_gpu_parity.py), fused step
1e-5, oracle 1e-3; bf16 — 1e-2 (stated tolerance: bf16 operands, fp32 atomics)."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils.rnn import pack_padded_sequence

from latex_ocr_b200 import _lib
from latex_ocr_b200.params import grad_view
from util import build_model, load_golden

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import ref_model as rm
    return rm


def _close(got, want, tol, name, floor=2e-8):
    """max-abs error below tol * max|want|, with an absolute floor for gradients that are pure rounding noise."""
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    assert torch.isfinite(got).all(), name
    err = (got - want).abs().max().item()
    assert err <= tol * want.abs().max().item() + floor, (name, err, want.abs().max().item())


def _check_summary(name, got, want, tol):
    """(copied from test_gpu_parity.py) golden gradients are stored whole or as {head, sum, abssum} summaries."""
    if isinstance(want, dict):
        g = got.reshape(-1)
        assert torch.isfinite(g).all(), name
        meanabs = want["abssum"] / g.numel()
        err = (g[:256].double().cpu() - want["head"].double()).abs().max().item()
        assert err <= tol * 5 * max(want["head"].abs().max().item(), meanabs) + 2e-8, (name, err)
        scale = want["abssum"] + 1e-30
        assert abs(g.double().sum().item() - want["sum"]) / scale < tol, name
        assert abs(g.double().abs().sum().item() - want["abssum"]) / scale < tol, name
    else:
        _close(got, want, tol, name)


def reference_get_loss(model, encoder_optimizer, decoder_optimizer, criterion, img, formula):
    """The body of the reference's Img2SeqModel.getLoss (img2seq_torch.py:136-172) on this package's modules.  The only
    edit: current torch's PackedSequence has four fields, so the packed data is taken with ``.data``."""
    img = img.to("cuda")
    formula = formula.to("cuda")
    imgs = model.encoder(img)
    scores, caps_sorted, decode_lengths, alphas, sort_ind = model.decoder(
        imgs, formula, torch.LongTensor([[len(i)] for i in formula]))
    targets = caps_sorted[:, 1:]
    scores = pack_padded_sequence(scores, decode_lengths, batch_first=True).data
    targets = pack_padded_sequence(targets, decode_lengths, batch_first=True).data
    loss = criterion(scores, targets)
    alpha_c = 1.
    loss += alpha_c * ((1. - alphas.sum(dim=1)) ** 2).mean()
    decoder_optimizer.zero_grad()
    if encoder_optimizer is not None:
        encoder_optimizer.zero_grad()
    loss.backward()
    decoder_optimizer.step()
    if encoder_optimizer is not None:
        encoder_optimizer.step()
    return -loss.item()


def _optimizers(m, lr=1e-3):
    return (torch.optim.Adam(m.encoder.parameters(), lr=lr), torch.optim.Adam(m.decoder.parameters(), lr=lr))


def custom_loss(preds, caps, decode_lengths, alphas):
    """Label-smoothed CE over the decoded positions + a regulariser whose weight changes with t (so d loss / d alpha does)."""
    B, T, V = preds.shape
    dev = preds.device
    act = (torch.arange(T, device=dev)[None, :] < torch.tensor(decode_lengths, device=dev)[:, None]).to(preds.dtype)
    lp = F.log_softmax(preds, dim=-1)
    nll = -lp.gather(2, caps[:, 1:T + 1].unsqueeze(2)).squeeze(2)
    ce = ((0.9 * nll - 0.1 * lp.mean(dim=2)) * act).sum() / act.sum()
    w = torch.linspace(0.5, 1.5, T, dtype=preds.dtype, device=dev)
    reg = ((1. - (alphas * w[None, :, None]).sum(dim=1)) ** 2).mean()
    return ce + 0.7 * reg


def _ragged_case(V=50, B=5, seed=3):
    rm = _oracle()
    pe, pd = rm.init_params(V, seed=seed)
    _, formula = rm.synthetic_batch(B, 32, 64, V, 3, 9, seed=seed + 1)
    lengths = torch.tensor([[10], [4], [7], [4], [9]])[:B]
    g = torch.Generator().manual_seed(seed + 2)
    enc = torch.randn(B, 4, 7, 512, generator=g) * 0.5
    return pe, pd, formula, lengths, enc


def _run_custom(m, formula, lengths, enc):
    x = enc.cuda().requires_grad_(True)
    preds, caps, dl, alphas, _ = m.decoder(x, formula.cuda(), lengths)
    custom_loss(preds, caps, dl, alphas).backward()
    return x.grad, {k: p.grad.detach().clone() for k, p in m.decoder.named_parameters()}


# 1 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny_eval", "tiny_nopos", "cfg1"])
def test_reference_get_loss_body_vs_golden(name):
    rm = _oracle()
    rec = load_golden(name)
    c = rec["case"]
    pe, pd = rm.init_params(c["V"], seed=c["pseed"])
    img, formula = rm.synthetic_batch(c["B"], c["H"], c["W"], c["V"], c["tmin"], c["tmax"], seed=c["dseed"])
    m = build_model(c["V"], pe, pd, "fp32", positional=c["positional"], train=c["train"])
    eo, do = _optimizers(m)
    neg = reference_get_loss(m, eo, do, nn.CrossEntropyLoss(), img, formula)
    assert abs(-neg - rec["loss"]) / abs(rec["loss"]) < 1e-4, (neg, rec["loss"])
    for k, p in m.decoder.named_parameters():
        if k == "attention.full_att.bias":
            assert p.grad.abs().max().item() < 1e-6        # exactly 0 (softmax shift invariance); rounding noise in the reference
            continue
        _check_summary("dec." + k, p.grad.float().cpu(), rec["grad_dec"][k], 1e-3)
    for k, p in m.encoder.named_parameters():
        _check_summary("enc." + k, p.grad.float().cpu(), rec["grad_enc"][k], 1e-3)


# 2 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_generic_backward_bit_identical_to_fused(precision):
    """Generic mode fed the fused loss's own d predictions and d alpha == the fused backward, bit for bit."""
    rm = _oracle()
    V = 70
    pe, pd = rm.init_params(V, seed=31)
    img, formula = rm.synthetic_batch(4, 32, 96, V, 6, 6, seed=32)
    m = build_model(V, pe, pd, precision, train=True, impl="tc" if precision == "bf16" else "simt")
    dec = m.decoder
    B, T = formula.shape[0], formula.shape[1] - 1
    with _lib.option(deterministic=1), torch.no_grad():
        enc = m.encoder.forward_raw(img.cuda(), need_grad=True)
        enc = enc.reshape(B, -1, enc.shape[3])
        R = enc.shape[1]
        caps = formula.cuda()
        dec.seed_dropout(1234)
        ws = dec.run_forward(enc, caps, [T] * B, with_loss=True, need_grad=True, dropout_mask="philox")
        dec.run_backward(ws)
        want_g = dec.store.grad.clone()
        want_denc = ws["t"]["denc"].clone()
        dlogits = ws["t"]["dlogits"].clone()                 # [B][T][ldl]: rows ldl apart
        dalpha = ws["t"]["dreg"][:, None, :].expand(B, T, R).contiguous()
        dec.store.grad.zero_()
        ws["t"]["denc"].zero_()
        dec.seed_dropout(1234)
        ws = dec.run_forward(enc, caps, [T] * B, with_loss=False, need_grad=True, dropout_mask="philox")
        a = ws["args"]
        a.dpred_ext, a.dpred_stride, a.dalpha_ext = dlogits.data_ptr(), dlogits.shape[2], dalpha.data_ptr()
        dec.run_backward(ws)
        torch.cuda.synchronize()
        assert torch.equal(dec.store.grad, want_g)
        assert torch.equal(ws["t"]["denc"], want_denc)


# 3 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 1e-2)])
def test_autograd_step_matches_fused_step(precision, tol):
    rm = _oracle()
    V = 64
    pe, pd = rm.init_params(V, seed=41)
    img, formula = rm.synthetic_batch(6, 48, 128, V, 10, 10, seed=42)
    impl = "tc" if precision == "bf16" else "simt"
    fused = build_model(V, pe, pd, precision, train=True, impl=impl)
    auto = build_model(V, pe, pd, precision, train=True, impl=impl)
    fused.decoder.seed_dropout(77)
    auto.decoder.seed_dropout(77)
    loss = fused.train_step(img.cuda(), formula.cuda(), sync=True)
    eo, do = _optimizers(auto)
    neg = reference_get_loss(auto, eo, do, nn.CrossEntropyLoss(), img, formula)
    assert abs(-neg - loss[0].item()) / loss[0].item() < max(tol, 1e-5)
    for mod in ("encoder", "decoder"):
        for k, p in getattr(auto, mod).named_parameters():
            q = dict(getattr(fused, mod).named_parameters())[k]
            if k == "attention.full_att.bias":
                continue
            _close(p.grad, q.grad, tol, mod + "." + k, floor=1e-9)
    # same Philox call counter afterwards: one call per step either way
    assert torch.equal(auto.decoder.dropout_state.cpu(), fused.decoder.dropout_state.cpu())


# 4, 5 ------------------------------------------------------------------------------------------------------------------------
def test_custom_loss_vs_cpu_oracle_ragged():
    rm = _oracle()
    V = 50
    pe, pd, formula, lengths, enc = _ragged_case(V)
    m = build_model(V, pe, pd, "fp32")
    dx, grads = _run_custom(m, formula, lengths, enc)
    pdd = {k: v.double().requires_grad_(True) for k, v in pd.items()}
    xd = enc.double().requires_grad_(True)
    preds, caps, dl, alphas, _ = rm.decoder_forward(pdd, xd, formula, lengths)
    custom_loss(preds, caps, dl, alphas).backward()
    assert dx.shape == enc.shape
    _close(dx, xd.grad, 1e-3, "d encoder_out")
    for k, g in grads.items():
        if k == "attention.full_att.bias":
            continue
        _close(g, pdd[k].grad, 1e-3, k)


@pytest.mark.parametrize("option", ["dec_cl_bwd", "dec_fuse_bwd", "att_bwd_mma", "att_maskbits"])
def test_custom_loss_under_backward_schedules(option):
    V = 50
    pe, pd, formula, lengths, enc = _ragged_case(V)
    L = _lib.lib()
    m = build_model(V, pe, pd, "bf16", impl="tc")
    want_dx, want = _run_custom(m, formula, lengths, enc)
    with _lib.option(**{option: 1 - L.lo_get_option(option.encode())}):
        m.decoder.zero_grad()
        dx, got = _run_custom(m, formula, lengths, enc)
    _close(dx, want_dx, 1e-2, "d encoder_out")
    for k in want:
        if k != "attention.full_att.bias":
            _close(got[k], want[k], 1e-2, k, floor=1e-7)


# 6 ---------------------------------------------------------------------------------------------------------------------------
def test_gradient_bookkeeping():
    rm = _oracle()
    V = 40
    pe, pd = rm.init_params(V, seed=51)
    img, formula = rm.synthetic_batch(3, 32, 64, V, 5, 5, seed=52)
    m = build_model(V, pe, pd, "fp32")
    lengths = torch.LongTensor([[formula.shape[1]]] * 3)
    params = list(m.encoder.named_parameters(prefix="encoder")) + list(m.decoder.named_parameters(prefix="decoder"))

    def step():
        preds, caps, dl, alphas, _ = m.decoder(m.encoder(img.cuda()), formula.cuda(), lengths)
        custom_loss(preds, caps, dl, alphas).backward()

    step()
    once = {k: p.grad.clone() for k, p in params}
    step()                                               # no zero_grad: accumulates
    for k, p in params:
        _close(p.grad, 2 * once[k], 1e-5, k, floor=1e-9)
    for set_to_none in (True, False):
        m.encoder.zero_grad(set_to_none=set_to_none)
        m.decoder.zero_grad(set_to_none=set_to_none)
        for k, p in params:
            assert (p.grad is None) if set_to_none else (p.grad.abs().max().item() == 0), k
        step()
        for k, p in params:
            _close(p.grad, once[k], 1e-5, k, floor=1e-9)
    # frozen parameters get no gradient
    m.encoder.fine_tune(False)
    m.decoder.fine_tune_embeddings(False)
    m.encoder.zero_grad(set_to_none=True)
    m.decoder.zero_grad(set_to_none=True)
    step()
    for k, p in params:
        assert (p.grad is None) == (not p.requires_grad), k
    assert m.encoder.cnn["0"].weight.grad is None and m.decoder.embedding.weight.grad is None
    # the fused step afterwards still leaves its gradients in p.grad
    m.encoder.fine_tune(True)
    m.decoder.fine_tune_embeddings(True)
    m.train_step(img.cuda(), formula.cuda(), sync=True)
    for mod in (m.encoder, m.decoder):
        for k, p in mod.named_parameters():
            assert p.grad is not None and torch.equal(p.grad, grad_view(mod.store, p)), k
        assert mod.store.grad.abs().sum().item() > 0


# 7 ---------------------------------------------------------------------------------------------------------------------------
def test_torch_optimizer_step_is_visible_to_the_next_forward():
    rm = _oracle()
    V = 48
    pe, pd = rm.init_params(V, seed=61)
    img, formula = rm.synthetic_batch(4, 32, 96, V, 7, 7, seed=62)
    m = build_model(V, pe, pd, "bf16", impl="tc")
    eo, do = _optimizers(m, lr=1e-2)
    reference_get_loss(m, eo, do, nn.CrossEntropyLoss(), img, formula)
    sd_e = {k: v.detach().cpu().clone() for k, v in m.encoder.state_dict().items()}
    sd_d = {k: v.detach().cpu().clone() for k, v in m.decoder.state_dict().items()}
    assert not torch.equal(sd_d["fc.weight"], pd["fc.weight"])
    fresh = build_model(V, sd_e, sd_d, "bf16", impl="tc")
    lengths = torch.LongTensor([[formula.shape[1]]] * 4)
    with torch.no_grad():
        outs = []
        for mm in (m, fresh):
            x = mm.encoder(img.cuda())
            preds, _, _, alphas, _ = mm.decoder(x, formula.cuda(), lengths)
            outs.append((x, preds, alphas))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# 8 ---------------------------------------------------------------------------------------------------------------------------
def test_backward_of_overwritten_forward_state_raises():
    V = 50
    pe, pd, formula, lengths, enc = _ragged_case(V)
    m = build_model(V, pe, pd, "fp32")
    x = enc.cuda().requires_grad_(True)
    first = m.decoder(x, formula.cuda(), lengths)
    m.decoder(x, formula.cuda(), lengths)              # same shape: overwrites the saved state of the first call
    with pytest.raises(_lib.LatexOcrB200Error):
        first[0].sum().backward()
    img, _ = _oracle().synthetic_batch(2, 32, 64, V, 3, 3, seed=5)
    y1 = m.encoder(img.cuda())
    m.encoder(img.cuda())
    with pytest.raises(_lib.LatexOcrB200Error):
        y1.sum().backward()


# 9 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_grad_enabled_forward_equals_no_grad_forward(precision):
    rm = _oracle()
    V = 45
    pe, pd = rm.init_params(V, seed=71)
    img, formula = rm.synthetic_batch(5, 32, 96, V, 3, 8, seed=72)
    lengths = torch.tensor([[9], [4], [7], [4], [6]])
    m = build_model(V, pe, pd, precision, train=True, impl="tc" if precision == "bf16" else "simt")
    outs = []
    for grad in (False, True):
        m.decoder.seed_dropout(5)
        with torch.set_grad_enabled(grad):
            x = m.encoder(img.cuda())
            res = m.decoder(x, formula.cuda(), lengths)
        assert (res[0].grad_fn is not None) == grad
        outs.append((x.detach().clone(), res[0].detach().clone(), res[1], res[2], res[3].detach().clone(), res[4]))
    for a, b in zip(*outs):
        assert a == b if isinstance(a, list) else torch.equal(a, b)


# 10 --------------------------------------------------------------------------------------------------------------------------
def test_dropout_replay_with_interleaved_forward():
    V = 50
    pe, pd, formula, lengths, enc = _ragged_case(V)
    m = build_model(V, pe, pd, "fp32", train=True)
    m.decoder.seed_dropout(99, call=3)
    want_dx, want = _run_custom(m, formula, lengths, enc)
    m.decoder.zero_grad(set_to_none=True)
    m.decoder.seed_dropout(99, call=3)
    x = enc.cuda().requires_grad_(True)
    preds, caps, dl, alphas, _ = m.decoder(x, formula.cuda(), lengths)
    other = m.decoder(enc[:3, :2].cuda(), formula[:3, :6].cuda(), torch.tensor([[6], [5], [6]]))   # another shape in between
    other[0].sum().backward()
    m.decoder.zero_grad(set_to_none=True)
    custom_loss(preds, caps, dl, alphas).backward()
    _close(x.grad, want_dx, 1e-5, "d encoder_out", floor=1e-9)
    for k, p in m.decoder.named_parameters():
        _close(p.grad, want[k], 1e-5, k, floor=1e-9)
