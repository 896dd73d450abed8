"""-m gpu: training the TensorFlow-flavour decoder through loss.backward() — autograd of tf_decoder.Decoder.train_outputs (and
Decoder.forward) on the CUDA kernels (lo_tfdec_backward in its generic mode), against the fp64 CPU restatement
oracle/ref_tf_model.py with autograd, the fused loss_and_backward / compute_gradients, and the bookkeeping rules of torch
(gradient accumulation, frozen parameters, optimizer visibility, stale saved state).  Tolerances: fp32 — oracle 1e-4 of each
tensor's max-abs (as test_gpu_tf_decoder.py), fused path 1e-5; bf16 — 6e-2 (the stated bound of the bf16 oracle test)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from latex_ocr_b200 import _lib
from latex_ocr_b200.params import grad_view
from util import Cfg, relerr

pytestmark = pytest.mark.gpu


def _cfg(**kw):
    return Cfg(attn_cell_config={"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}, max_length_formula=10, **kw)


def _setup(V=40, N=3, R=21, T=7, seed=3, precision="fp32", impl="simt", **kw):
    from latex_ocr_b200.tf_decoder import Decoder
    from oracle import ref_tf_model as tfm
    g = torch.Generator().manual_seed(seed)
    p = tfm.init_params_tf(V, seed=seed)
    p["y_W_o"] = p["y_W_o"] * 4.0
    enc = torch.relu(torch.randn(N, R, 512, generator=g)) * 0.7
    formula = torch.randint(0, V, (N, T), generator=g)
    dec = Decoder(_cfg(**kw), V, V - 1, device="cuda", precision=precision, impl=impl)
    dec.load_tf_variables(p)
    return tfm, p, dec, enc, formula


def _keeps(N, T, seed=11, kp=0.8):
    g = torch.Generator().manual_seed(seed)
    kh = (torch.rand(N, T, 512, generator=g) < kp).float() / kp
    ko = (torch.rand(N, T, 512, generator=g) < kp).float() / kp
    return kh, ko


def custom_loss(logits, alphas, formula, lengths):
    """Label-smoothed CE over the valid tokens of ragged lengths + a regulariser on alphas whose weight changes with t (so
    d loss / d alpha does too).  ``alphas`` None: the CE alone."""
    N, T, V = logits.shape
    dev = logits.device
    act = (torch.arange(T, device=dev)[None, :] < lengths.to(dev)[:, None]).to(logits.dtype)
    lp = F.log_softmax(logits, dim=-1)
    nll = -lp.gather(2, formula.to(dev).unsqueeze(2)).squeeze(2)
    ce = ((0.9 * nll - 0.1 * lp.mean(dim=2)) * act).sum() / act.sum()
    if alphas is None:
        return ce
    w = torch.linspace(0.5, 1.5, T, dtype=logits.dtype, device=dev)
    return ce + 0.7 * ((1. - (alphas * w[None, :, None]).sum(dim=1)) ** 2).mean()


def _oracle(tfm, p, enc, formula, lengths, keep_h=None, keep_o=None, with_alphas=True):
    p = {k: v.clone().double().requires_grad_(True) for k, v in p.items()}
    enc = enc.clone().double().requires_grad_(True)
    kh = None if keep_h is None else keep_h.double()
    ko = None if keep_o is None else keep_o.double()
    logits, alphas = tfm.decoder_train_logits(p, enc, formula, kh, ko)
    custom_loss(logits, alphas if with_alphas else None, formula, lengths).backward()
    return logits.detach(), alphas.detach(), {k: v.grad for k, v in p.items()}, enc.grad


def _check_all(dec, got_dx, want_dx, want_grads, tol):
    assert relerr(got_dx.reshape(want_dx.shape), want_dx) < tol, "d enc"
    for k, q in dec.named_parameters():
        assert q.grad is not None, k
        assert relerr(q.grad, want_grads[k].reshape(q.grad.shape)) < tol, k


# 1, 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl,tol", [("fp32", "simt", 1e-4), ("bf16", "tc", 6e-2)])
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("layout", ["NRC", "NHWC"])
def test_custom_loss_vs_oracle(precision, impl, tol, dropout, layout):
    tfm, p, dec, enc, formula = _setup(N=4, R=21, T=9, precision=precision, impl=impl)
    N, T = formula.shape
    lengths = torch.tensor([9, 6, 3, 7])
    kh, ko = _keeps(N, T) if dropout else (None, None)
    want_lg, want_al, want_g, want_dx = _oracle(tfm, p, enc, formula, lengths, kh, ko)
    x = (enc if layout == "NRC" else enc.view(N, 3, 7, 512)).cuda().requires_grad_(True)
    dec.zero_grad(set_to_none=True)
    logits, alphas = dec.train_outputs(x, formula.cuda(), kh, ko)
    assert logits.shape == (N, T, 40) and alphas.shape == (N, T, 21)
    assert relerr(logits, want_lg) < tol and relerr(alphas, want_al) < tol
    custom_loss(logits, alphas, formula, lengths).backward()
    assert x.grad.shape == x.shape and x.grad.dtype == x.dtype
    _check_all(dec, x.grad, want_dx, want_g, tol)


# 3 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dropout", [False, True])
def test_masked_ce_through_autograd_equals_fused(dropout):
    tfm, p, dec, enc, formula = _setup(seed=4)
    N, T = formula.shape
    lengths = torch.tensor([7, 2, 5])
    kh, ko = _keeps(N, T, seed=13) if dropout else (None, None)
    x = enc.cuda()
    l, de = dec.loss_and_backward(x, formula.cuda(), lengths, kh, ko)
    fused = {k: q.grad.clone() for k, q in dec.named_parameters()}
    de, l = de.clone(), l.clone()
    dec.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    logits, _ = dec.train_outputs(xg, formula.cuda(), kh, ko)
    loss = tfm.masked_ce(logits, formula.cuda(), lengths)[0]
    assert abs(loss.item() - l[0].item()) <= 1e-5 * abs(l[0].item())
    loss.backward()
    assert relerr(xg.grad, de) < 1e-5
    for k, q in dec.named_parameters():
        assert relerr(q.grad, fused[k]) < 1e-5, k


# 4 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,impl", [("fp32", "simt"), ("bf16", "tc")])
def test_grad_enabled_outputs_equal_no_grad_outputs(precision, impl):
    tfm, p, dec, enc, formula = _setup(seed=6, precision=precision, impl=impl)
    kh, ko = _keeps(*formula.shape, seed=17)
    x, f = enc.cuda(), formula.cuda()
    outs = []
    for grad in (False, True):
        with torch.set_grad_enabled(grad):
            lg, al = dec.train_outputs(x, f, kh, ko)
        assert (lg.grad_fn is not None) == grad and (al.grad_fn is not None) == grad
        outs.append((lg.detach().clone(), al.detach().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(dec.train_logits(x, f, kh, ko), outs[1][0])
    train, _ = dec(x, f, 1.0)
    assert train.grad_fn is not None and torch.equal(train.detach(), dec.train_logits(x, f))


# 5 ---------------------------------------------------------------------------------------------------------------------------
def test_gradient_bookkeeping():
    tfm, p, dec, enc, formula = _setup(seed=8)
    lengths = torch.tensor([7, 4, 6])
    x, f = enc.cuda(), formula.cuda()

    def step():
        logits, alphas = dec.train_outputs(x, f)
        custom_loss(logits, alphas, formula, lengths).backward()

    dec.zero_grad(set_to_none=True)
    step()
    once = {k: q.grad.clone() for k, q in dec.named_parameters()}
    step()                                               # no zero_grad: accumulates
    for k, q in dec.named_parameters():
        assert relerr(q.grad, 2 * once[k]) < 1e-5, k
    for set_to_none in (True, False):
        dec.zero_grad(set_to_none=set_to_none)
        for k, q in dec.named_parameters():
            assert (q.grad is None) if set_to_none else (q.grad.abs().max().item() == 0), k
        step()
        for k, q in dec.named_parameters():
            assert relerr(q.grad, once[k]) < 1e-5, k
    # frozen parameters get no gradient
    dec.embedding_table.requires_grad_(False)
    dec.lstm.kernel.requires_grad_(False)
    dec.zero_grad(set_to_none=True)
    step()
    for k, q in dec.named_parameters():
        assert (q.grad is None) == (not q.requires_grad), k
    assert dec.embedding_table.grad is None and dec.lstm.kernel.grad is None
    # the fused path afterwards leaves its gradients in p.grad again
    dec.embedding_table.requires_grad_(True)
    dec.lstm.kernel.requires_grad_(True)
    dec.loss_and_backward(x, f, lengths)
    for k, q in dec.named_parameters():
        assert q.grad is not None and torch.equal(q.grad, grad_view(dec.store, q)), k
    assert dec.store.grad.abs().sum().item() > 0


# 6 ---------------------------------------------------------------------------------------------------------------------------
def test_torch_optimizer_step_is_visible_to_the_next_forward():
    from latex_ocr_b200.tf_decoder import Decoder
    tfm, p, dec, enc, formula = _setup(seed=9, precision="bf16", impl="tc")
    lengths = torch.tensor([7, 5, 7])
    x, f = enc.cuda(), formula.cuda()
    opt = torch.optim.Adam(dec.parameters(), lr=1e-2)
    logits, alphas = dec.train_outputs(x, f)
    opt.zero_grad()
    custom_loss(logits, alphas, formula, lengths).backward()
    opt.step()
    sd = {k: v.detach().clone() for k, v in dec.state_dict().items()}
    assert not torch.equal(sd["y_W_o"].cpu(), p["y_W_o"])
    fresh = Decoder(_cfg(), 40, 39, device="cuda", precision="bf16", impl="tc")
    fresh.load_state_dict(sd)
    with torch.no_grad():
        a = dec.train_outputs(x, f)
        b = fresh.train_outputs(x, f)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# 7 ---------------------------------------------------------------------------------------------------------------------------
def test_backward_of_overwritten_forward_state_raises():
    tfm, p, dec, enc, formula = _setup(seed=10)
    x = enc.cuda().requires_grad_(True)
    first = dec.train_outputs(x, formula.cuda())
    dec.train_outputs(x, formula.cuda())                # same shape: overwrites the saved state of the first call
    with pytest.raises(_lib.LatexOcrB200Error):
        first[0].sum().backward()


# 8 ---------------------------------------------------------------------------------------------------------------------------
def test_forward_with_greedy_decode_of_the_same_length():
    """Decoder.forward = teacher-forced pass + decode(); with T == max_length_formula + 2 both have the same shape, and the decode
    must not overwrite the state the backward needs."""
    tfm, p, dec, enc, formula = _setup(seed=12, T=12, decoding="greedy")
    assert formula.shape[1] == dec.max_length_formula + 2
    N = formula.shape[0]
    lengths = torch.tensor([12, 8, 5])
    _, _, want_g, want_dx = _oracle(tfm, p, enc, formula, lengths, with_alphas=False)
    x = enc.cuda().requires_grad_(True)
    dec.zero_grad(set_to_none=True)
    train, test = dec(x, formula.cuda(), 1.0)
    assert test.ids.shape[0] == N
    custom_loss(train, None, formula, lengths).backward()
    _check_all(dec, x.grad, want_dx, want_g, 1e-4)
    # with dropout: masks drawn inside forward, reused by the backward
    dec.zero_grad(set_to_none=True)
    train, _ = dec(x, formula.cuda(), 0.7)
    custom_loss(train, None, formula, lengths).backward()
    assert all(torch.isfinite(q.grad).all() for q in dec.parameters())


# 9 ---------------------------------------------------------------------------------------------------------------------------
def _tf_model(precision, impl, V=30):
    from latex_ocr_b200.data import SimpleVocab
    from latex_ocr_b200.img2seq_tf import Img2SeqModel
    torch.manual_seed(21)
    cfg = _cfg(batch_size=3, decoding="greedy", dropout=1.0, lr_init=1e-3)
    return Img2SeqModel(cfg, vocab=SimpleVocab(V), device="cuda", precision=precision, impl=impl).build_train(cfg)


def _tf_batch(V=30, N=3, T=6, seed=22):
    rng = np.random.RandomState(seed)
    img = np.full((N, 1, 32, 64), 255, np.uint8)
    ink = rng.rand(N, 1, 32, 64) < 0.1
    img[ink] = rng.randint(0, 255, int(ink.sum()))
    formula = rng.randint(0, V - 3, (N, T)).astype(np.int64)
    lengths = np.array([T, T - 2, 3], np.int32)
    for b, n in enumerate(lengths):
        formula[b, n - 1] = V - 1                                   # END, then PAD
        formula[b, n:] = V - 2
    return torch.from_numpy(img).cuda(), formula, lengths


def test_end_to_end_autograd_equals_compute_gradients():
    from oracle import ref_tf_model as tfm
    m = _tf_model("fp32", "simt")
    img, formula, lengths = _tf_batch()
    m.compute_gradients(img, (formula, lengths))
    fused = {(mod, k): q.grad.clone() for mod in (m.encoder, m.decoder) for k, q in mod.named_parameters()}
    for mod in (m.encoder, m.decoder):
        mod.zero_grad(set_to_none=True)
    f = torch.from_numpy(formula).cuda()
    enc = m.encoder(img)
    logits, _ = m.decoder.train_outputs(enc, f)
    tfm.masked_ce(logits, f, torch.from_numpy(lengths).long())[0].backward()
    for (mod, k), want in fused.items():
        got = dict(mod.named_parameters())[k].grad
        assert relerr(got, want) < 1e-5, k


def test_torch_adam_steps_reduce_the_loss_bf16():
    from oracle import ref_tf_model as tfm
    m = _tf_model("bf16", "tc")
    img, formula, lengths = _tf_batch(seed=23)
    f, lens = torch.from_numpy(formula).cuda(), torch.from_numpy(lengths).long()
    opt = torch.optim.Adam(list(m.encoder.parameters()) + list(m.decoder.parameters()), lr=1e-3)
    losses = []
    for _ in range(12):
        opt.zero_grad()
        logits, _ = m.decoder.train_outputs(m.encoder(img), f)
        loss = tfm.masked_ce(logits, f, lens)[0]
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and losses[-1] < 0.9 * losses[0], losses
