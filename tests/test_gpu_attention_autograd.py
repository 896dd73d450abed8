"""-m gpu: training through the stand-alone Attention module — autograd of Attention.forward on lo_attention_step_backward (one
pass of the TMA-ring attention backward that also writes d att1, then the encoder_att / decoder_att GEMMs).  Checked against a
float64 restatement of the kernel's own inputs, the fp64 oracle module under torch autograd, the fused DecoderWithAttention
autograd (the reference's per-step loop restated on dec.attention) and the bookkeeping rules of torch.  Tolerances: kernel 1e-5
of max-abs (bf16 d att1: one bf16 ulp of the float64 value rounded to bf16, plus that 1e-5); fp32 module 1e-5 on outputs, 1e-4
on gradients; reference loop 1e-4 on outputs, 1e-3 on gradients; bf16 + wgmma module: the bounds below, set from the measured
error."""
import pytest
import torch
import torch.nn.functional as F

from latex_ocr_b200 import _lib
from latex_ocr_b200.decoder import Attention, DecoderWithAttention
from latex_ocr_b200.params import grad_view
from util import build_model

pytestmark = pytest.mark.gpu

# bf16 storage + wgmma GEMMs against the fp64 oracle, max-abs error over max-abs value, measured on an H100 for the three losses
# below: outputs 2.2e-3, gradients 0.20-0.21 (bf16 enc, att1 and weights in the forward move ReLU masks and softmax weights; the
# kernel's own share is checked at 1e-5 on its own inputs by test_step_kernel_vs_float64).  The bounds leave room for other seeds.
BF16_OUT_BOUND = 1e-2
BF16_GRAD_BOUND = 0.3
GRAD_NAMES = Attention._GRAD_NAMES


def _oracle():
    from oracle import ref_model as rm
    return rm


def _err(got, want):
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    assert torch.isfinite(got).all()
    return (got - want).abs().max().item() / max(want.abs().max().item(), 1e-30)


def _close(got, want, tol, name, floor=2e-8):
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    assert torch.isfinite(got).all(), name
    err = (got - want).abs().max().item()
    assert err <= tol * want.abs().max().item() + floor, (name, err, want.abs().max().item())


# 1 ---------------------------------------------------------------------------------------------------------------------------
def _kernel_inputs(B, R, A, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    enc = (torch.randn(B, R, A, generator=g, device=dev) * 0.5).to(dtype)
    att1 = (torch.randn(B, R, A, generator=g, device=dev) * 0.3).to(dtype)
    att2 = torch.randn(B, A, generator=g, device=dev) * 0.3
    wf = torch.rand(A, generator=g, device=dev) - 0.5
    e = (torch.relu(att1.double() + att2.double()[:, None, :]) * wf.double()).sum(2)
    alpha = torch.softmax(e, dim=1).float()
    ctx = (alpha.double()[:, :, None] * enc.double()).sum(1).float()
    dctx = torch.randn(B, A, generator=g, device=dev)
    dalpha = torch.randn(B, R, generator=g, device=dev) * 0.1
    return enc, att1, att2, wf, alpha, ctx, dctx, dalpha


def _reference64(enc, att1, att2, wf, alpha, ctx, dctx, dalpha):
    enc, att1, att2, wf, alpha, ctx, dctx = (t.double() for t in (enc, att1, att2, wf, alpha, ctx, dctx))
    dal = dalpha.double() if dalpha is not None else torch.zeros_like(alpha)
    s = (dctx * ctx).sum(1) + (alpha * dal).sum(1)
    de = alpha * (torch.einsum("brc,bc->br", enc, dctx) + dal - s[:, None])
    pre = att1 + att2[:, None, :]
    on = (pre > 0).double()
    datt1 = wf * de[:, :, None] * on
    datt2 = wf * (de[:, :, None] * on).sum(1)
    dwf = (de[:, :, None] * torch.relu(pre)).sum((0, 1))
    return de, datt1, datt2, dwf


def _step_backward(enc, att1, att2, wf, alpha, ctx, dctx, dalpha, D=64, impl=_lib.LO_IMPL_SIMT):
    """The kernel's own outputs (de, d att1, d att2, d full_att.weight) of lo_attention_step_backward."""
    L = _lib.lib()
    B, R, A = att1.shape
    dt = _lib.dt_of(enc)
    dev = enc.device
    h = torch.zeros(B, D, device=dev)
    w_enc = torch.zeros(A, A, dtype=enc.dtype, device=dev)
    w_dec = torch.zeros(A, D, dtype=enc.dtype, device=dev)
    de = torch.empty(B, R, device=dev)
    datt2 = torch.empty(B, A, device=dev)
    datt1 = torch.empty(B, R, A, dtype=enc.dtype, device=dev)
    gwf = torch.empty(A, device=dev)
    work = torch.zeros(L.lo_attention_step_workspace_bytes(B, R, A, A, dt), dtype=torch.uint8, device=dev)
    P = _lib.ptr
    _lib.check(L.lo_attention_step_backward(P(enc), P(att1), dt, P(h), P(att2), P(w_enc), P(w_dec), P(wf), P(alpha), P(ctx), P(dctx),
                                            P(dalpha), None, None, None, None, None, None, P(gwf), None, P(de), P(datt2), P(datt1),
                                            B, R, A, A, D, impl, P(work), _lib.stream_ptr()))
    return de, datt1, datt2, gwf


KERNEL_CASES = [(A, R, B) for A in (256, 512, 1024) for R, B in ((44, 5), (101, 3))] + [(512, 868, 64), (256, 868, 16), (1024, 868, 8)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("A,R,B", KERNEL_CASES)
def test_step_kernel_vs_float64(dtype, A, R, B):
    enc, att1, att2, wf, alpha, ctx, dctx, dalpha = _kernel_inputs(B, R, A, dtype, seed=A + R + B)
    de, datt1, datt2, gwf = _step_backward(enc, att1, att2, wf, alpha, ctx, dctx, dalpha)
    torch.cuda.synchronize()
    r_de, r_datt1, r_datt2, r_dwf = _reference64(enc, att1, att2, wf, alpha, ctx, dctx, dalpha)
    _close(de, r_de, 1e-5, "de")
    _close(datt2, r_datt2, 1e-5, "datt2")
    _close(gwf, r_dwf, 1e-5, "d full_att.weight")
    if dtype == torch.float32:
        _close(datt1, r_datt1, 1e-5, "datt1")
    else:
        _close_bf16(datt1, r_datt1)


def _close_bf16(got, want64):
    """The kernel rounds its fp32 value (within 1e-5 of max-abs, like de) to bf16: at most that plus one bf16 ulp from the
    float64 value rounded to bf16."""
    want = want64.to(torch.bfloat16).double()
    ulp = torch.where(want != 0, 2.0 ** (torch.floor(torch.log2(want.abs().clamp_min(1e-38))) - 7), torch.zeros_like(want))
    slack = 1e-5 * want64.abs().max().item()
    assert ((got.double() - want).abs() <= ulp + slack).all(), "d att1 beyond one bf16 ulp"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("A,R,B", [(512, 868, 64), (256, 101, 3), (1024, 44, 5)])
def test_step_kernel_shares_the_attention_backward_arithmetic(dtype, A, R, B):
    """de and d att2 bit for bit those of lo_attention_backward on the same inputs: the d att1 variant changed no shared sum."""
    L = _lib.lib()
    enc, att1, att2, wf, alpha, ctx, dctx, _ = _kernel_inputs(B, R, A, dtype, seed=7 * A + R)
    de, _, datt2, _ = _step_backward(enc, att1, att2, wf, alpha, ctx, dctx, None)
    de2 = torch.empty_like(de)
    datt2b = torch.empty_like(datt2)
    work = torch.zeros(L.lo_attention_workspace_bytes(B, A), dtype=torch.uint8, device="cuda")
    P = _lib.ptr
    _lib.check(L.lo_attention_backward(P(att1), P(enc), _lib.dt_of(enc), P(att2), None, A, P(wf), P(alpha), R, P(ctx), P(dctx), A, None,
                                       0, None, 0, P(de2), P(datt2b), None, A, None, None, None, B, R, A, A, P(work),
                                       _lib.stream_ptr()))
    assert torch.equal(de, de2) and torch.equal(datt2, datt2b)


def _check_vs_float64(dtype, A, R, B, seed):
    enc, att1, att2, wf, alpha, ctx, dctx, dalpha = _kernel_inputs(B, R, A, dtype, seed=seed)
    outs = _step_backward(enc, att1, att2, wf, alpha, ctx, dctx, dalpha)
    torch.cuda.synchronize()
    ref = _reference64(enc, att1, att2, wf, alpha, ctx, dctx, dalpha)
    for name, got, want in zip(("de", "datt1", "datt2", "d full_att.weight"), outs, ref):
        if name == "datt1" and dtype == torch.bfloat16:
            _close_bf16(got, want)
        else:
            _close(got, want, 1e-5, name)
    return outs


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("A,R,B,opts", [(1024, 12, 136, {}), (512, 44, 5, {"att_cluster": 0}), (1024, 44, 5, {"att_cluster": 0})],
                         ids=["one-split", "no-cluster-512", "no-cluster-1024"])
def test_step_kernel_without_cluster(dtype, A, R, B, opts):
    """The non-cluster launches of the d att1 kernel: B >= 133 gives one split per batch row; att_cluster=0 gives several splits
    whose d w_full partials meet with atomics.  With "deterministic" the splits of a row are folded into one (fixed order) and two
    calls give the same bits."""
    with _lib.option(**opts):
        _check_vs_float64(dtype, A, R, B, seed=3 * A + B)
        with _lib.option(deterministic=1):
            first = _check_vs_float64(dtype, A, R, B, seed=5 * A + B)
            second = _check_vs_float64(dtype, A, R, B, seed=5 * A + B)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


def test_d_att1_is_not_written_when_nothing_reads_it():
    """denc, the encoder_att gradients and datt1 all NULL: the workspace's d att1 region keeps its sentinel; asking for d enc
    overwrites it."""
    L = _lib.lib()
    B, R, A, D = 5, 44, 512, 64
    enc, att1, att2, wf, alpha, ctx, dctx, dalpha = _kernel_inputs(B, R, A, torch.bfloat16, seed=21)
    dt = _lib.LO_BF16
    h = torch.randn(B, D, device="cuda")
    w_enc = torch.randn(A, A, device="cuda").bfloat16()
    w_dec = torch.randn(A, D, device="cuda").bfloat16()

    def al(n):
        return (n + 255) // 256 * 256
    off = al(L.lo_attention_workspace_bytes(B, A)) + al(B * A * 4) + al(B * R * 4) + al(B * A * 4) + al(B * 4)
    n1 = B * R * A * 2
    work = torch.zeros(L.lo_attention_step_workspace_bytes(B, R, A, A, dt), dtype=torch.uint8, device="cuda")
    work[off:off + n1].fill_(0x5A)
    dh = torch.empty(B, D, device="cuda")
    gwd = torch.empty(A, D, device="cuda")
    gwf = torch.empty(A, device="cuda")
    denc = torch.empty(B, R, A, device="cuda")
    P = _lib.ptr

    def call(denc_):
        _lib.check(L.lo_attention_step_backward(P(enc), P(att1), dt, P(h), P(att2), P(w_enc), P(w_dec), P(wf), P(alpha), P(ctx),
                                                P(dctx), P(dalpha), P(denc_), P(dh), None, None, P(gwd), None, P(gwf), None, None,
                                                None, None, B, R, A, A, D, _lib.LO_IMPL_TC, P(work), _lib.stream_ptr()))
        torch.cuda.synchronize()
    call(None)
    assert (work[off:off + n1] == 0x5A).all()
    call(denc)
    assert not (work[off:off + n1] == 0x5A).all()


@pytest.mark.parametrize("impl,dtype,A,R,B", [("tc", torch.bfloat16, 512, 101, 3), ("tc", torch.bfloat16, 512, 868, 16),
                                              ("tc", torch.bfloat16, 256, 44, 5), ("tc", torch.bfloat16, 1024, 101, 3),
                                              ("simt", torch.bfloat16, 512, 101, 3), ("simt", torch.float32, 512, 101, 3)])
def test_step_gemms_vs_float64(impl, dtype, A, R, B):
    """The GEMMs after the kernel (on wgmma for bf16 + tc) against float64 of their own operands — the d att1 and d att2 the
    kernel returned, enc, h and the weights as stored: d enc = alpha (x) dctx + datt1 W_enc, d W_enc = datt1^T enc,
    d b_enc = colsum(datt1), d h = datt2 W_dec, d W_dec = datt2^T h, d b_dec = colsum(datt2)."""
    L = _lib.lib()
    D = 256
    enc, att1, att2, wf, alpha, ctx, dctx, dalpha = _kernel_inputs(B, R, A, dtype, seed=13 * A + R)
    g = torch.Generator(device="cuda").manual_seed(17)
    h = torch.randn(B, D, generator=g, device="cuda")
    w_enc = (torch.randn(A, A, generator=g, device="cuda") / A ** 0.5).to(dtype)
    w_dec = (torch.randn(A, D, generator=g, device="cuda") / D ** 0.5).to(dtype)
    dt = _lib.dt_of(enc)
    f = dict(denc=(B, R, A), dh=(B, D), gwe=(A, A), gbe=(A,), gwd=(A, D), gbd=(A,), datt2=(B, A))
    o = {k: torch.empty(s, device="cuda") for k, s in f.items()}
    datt1 = torch.empty(B, R, A, dtype=dtype, device="cuda")
    work = torch.zeros(L.lo_attention_step_workspace_bytes(B, R, A, A, dt), dtype=torch.uint8, device="cuda")
    P = _lib.ptr
    _lib.check(L.lo_attention_step_backward(P(enc), P(att1), dt, P(h), P(att2), P(w_enc), P(w_dec), P(wf), P(alpha), P(ctx), P(dctx),
                                            P(dalpha), P(o["denc"]), P(o["dh"]), P(o["gwe"]), P(o["gbe"]), P(o["gwd"]), P(o["gbd"]),
                                            None, None, None, P(o["datt2"]), P(datt1), B, R, A, A, D,
                                            _lib.LO_IMPL_TC if impl == "tc" else _lib.LO_IMPL_SIMT, P(work), _lib.stream_ptr()))
    torch.cuda.synchronize()
    d1 = datt1.double().reshape(B * R, A)
    d2 = o["datt2"].double()
    e = enc.double().reshape(B * R, A)
    want = {"denc": (alpha.double()[:, :, None] * dctx.double()[:, None, :]).reshape(B * R, A) + d1 @ w_enc.double(),
            "gwe": d1.t() @ e, "gbe": d1.sum(0), "dh": d2 @ w_dec.double(), "gwd": d2.t() @ h.double(), "gbd": d2.sum(0)}
    for k, w in want.items():
        _close(o[k], w, 1e-5, k)


# 2 ---------------------------------------------------------------------------------------------------------------------------
def _module_case(precision, seed=5, B=6, R=44, C=512, D=512):
    torch.manual_seed(seed)
    att = Attention(C, D, C, precision=precision)
    g = torch.Generator().manual_seed(seed + 1)
    enc = torch.randn(B, R, C, generator=g) * 0.5
    h = torch.randn(B, D, generator=g)
    gc = torch.randn(B, C, generator=g)
    ga = torch.randn(B, R, generator=g)
    return att, enc, h, gc, ga


def _loss(ctx, alpha, gc, ga, which):
    if which == "ctx":
        return (ctx * gc).sum()
    if which == "alpha":
        return (alpha * ga).sum()
    return (ctx * gc).sum() + (alpha * ga).sum()


@pytest.mark.parametrize("which", ["both", "ctx", "alpha"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_module_vs_oracle(precision, which):
    rm = _oracle()
    att, enc, h, gc, ga = _module_case(precision)
    p = {"attention." + k: v.detach().double().cpu().requires_grad_(True) for k, v in att.state_dict().items()}
    e64, h64 = enc.double().requires_grad_(True), h.double().requires_grad_(True)
    c64, a64 = rm.attention_forward(p, e64, h64)
    _loss(c64, a64, gc.double(), ga.double(), which).backward()

    x, y = enc.cuda().requires_grad_(True), h.cuda().requires_grad_(True)
    att.zero_grad(set_to_none=True)
    ctx, alpha = att(x, y)
    _loss(ctx, alpha, gc.cuda(), ga.cuda(), which).backward()
    got = [("d enc", x.grad, e64.grad), ("d h", y.grad, h64.grad)] + \
          [(n, dict(att.named_parameters())[n].grad, p["attention." + n].grad) for n in GRAD_NAMES if n != "full_att.bias"]
    assert att.full_att.bias.grad is not None and att.full_att.bias.grad.abs().max().item() == 0.0   # sum_r de_r = 0 exactly
    if precision == "fp32":
        _close(ctx, c64, 1e-5, "ctx")
        _close(alpha, a64, 1e-5, "alpha")
        for name, g_, w in got:
            _close(g_, w, 1e-4, name)
    else:
        out = max(_err(ctx, c64), _err(alpha, a64))
        errs = {name: _err(g_, w) for name, g_, w in got}
        print("bf16 + wgmma vs fp64 oracle (%s loss): outputs %.3e, gradients %s" % (which, out, errs))
        assert out <= BF16_OUT_BOUND and max(errs.values()) <= BF16_GRAD_BOUND, (out, errs)


# 3 ---------------------------------------------------------------------------------------------------------------------------
def reference_loop(dec, encoder_out, encoded_captions, caption_lengths):
    """DecoderWithAttention.forward of the reference (seq2seq_torch.py:267-320) in eval mode, restated on ``dec``'s parameter
    views and its ``dec.attention``: a per-step Python loop with a shrinking batch_size_t."""
    B, C = encoder_out.size(0), encoder_out.size(-1)
    enc = encoder_out.reshape(B, -1, C)
    R = enc.size(1)
    caption_lengths, sort_ind = caption_lengths.squeeze(1).sort(dim=0, descending=True)
    sort_ind = sort_ind.to(enc.device)
    enc = enc[sort_ind]
    caps = encoded_captions[sort_ind]
    emb = F.embedding(caps, dec.embedding.weight)
    mean = enc.mean(dim=1)
    h = F.linear(mean, dec.init_h.weight, dec.init_h.bias)
    c = F.linear(mean, dec.init_c.weight, dec.init_c.bias)
    decode_lengths = (caption_lengths - 1).tolist()
    T, V = max(decode_lengths), dec.vocab_size
    preds = torch.zeros(B, T, V, device=enc.device)
    alphas = torch.zeros(B, T, R, device=enc.device)
    ds = dec.decode_step
    for t in range(T):
        bt = sum(l > t for l in decode_lengths)
        ctx, alpha = dec.attention(enc[:bt], h[:bt])
        gate = torch.sigmoid(F.linear(h[:bt], dec.f_beta.weight, dec.f_beta.bias))
        h, c = torch._VF.lstm_cell(torch.cat([emb[:bt, t, :], gate * ctx], dim=1), (h[:bt], c[:bt]), ds.weight_ih, ds.weight_hh,
                                   ds.bias_ih, ds.bias_hh)
        preds[:bt, t, :] = F.linear(h, dec.fc.weight, dec.fc.bias)
        alphas[:bt, t, :] = alpha
    return preds, caps, decode_lengths, alphas, sort_ind


def smoothed_loss(preds, caps, decode_lengths, alphas):
    B, T, V = preds.shape
    act = (torch.arange(T, device=preds.device)[None, :] < torch.tensor(decode_lengths, device=preds.device)[:, None]).float()
    lp = F.log_softmax(preds, dim=-1)
    nll = -lp.gather(2, caps[:, 1:T + 1].unsqueeze(2)).squeeze(2)
    ce = ((0.9 * nll - 0.1 * lp.mean(dim=2)) * act).sum() / act.sum()
    w = torch.linspace(0.5, 1.5, T, device=preds.device)
    return ce + 0.7 * ((1. - (alphas * w[None, :, None]).sum(dim=1)) ** 2).mean()


def test_reference_loop_equals_fused_decoder():
    rm = _oracle()
    V = 50
    _, pd = rm.init_params(V, seed=3)
    _, formula = rm.synthetic_batch(5, 32, 64, V, 3, 9, seed=4)
    lengths = torch.tensor([[10], [4], [7], [4], [9]])
    enc = torch.randn(5, 4, 7, 512, generator=torch.Generator().manual_seed(5)) * 0.5
    dec = DecoderWithAttention(512, 512, 512, V, 512, precision="fp32")
    dec.load_state_dict(pd)
    dec.eval()
    caps = formula.cuda()
    runs = []
    for fn in (dec, lambda *a: reference_loop(dec, *a)):
        dec.zero_grad(set_to_none=True)
        x = enc.cuda().requires_grad_(True)
        preds, caps_s, dl, alphas, _ = fn(x, caps, lengths)
        smoothed_loss(preds, caps_s, dl, alphas).backward()
        runs.append((preds.detach(), alphas.detach(), x.grad, {k: p.grad.clone() for k, p in dec.named_parameters()}))
    (p0, a0, dx0, g0), (p1, a1, dx1, g1) = runs
    _close(p1, p0, 1e-4, "predictions")
    _close(a1, a0, 1e-4, "alphas")
    _close(dx1, dx0, 1e-3, "d encoder_out")
    for k in g0:
        _close(g1[k], g0[k], 1e-3, k)


# 4 ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_outputs_bitwise_equal_no_grad(precision):
    att, enc, h, _, _ = _module_case(precision)
    x, y = enc.cuda(), h.cuda()
    with torch.no_grad():
        c0, a0 = att(x, y)
    c1, a1 = att(x.requires_grad_(True), y)
    assert c1.grad_fn is not None and a1.grad_fn is not None
    assert c0.grad_fn is None
    assert torch.equal(c0, c1) and torch.equal(a0, a1)


def test_gradients_accumulate_and_zero_grad_and_frozen():
    att, enc, h, gc, ga = _module_case("fp32")
    x, y = enc.cuda(), h.cuda().requires_grad_(True)
    gc, ga = gc.cuda(), ga.cuda()
    att.zero_grad(set_to_none=True)
    _loss(*att(x, y), gc, ga, "both").backward()
    g1 = {n: p.grad.clone() for n, p in att.named_parameters()}
    dh1 = y.grad.clone()
    _loss(*att(x, y), gc, ga, "both").backward()
    for n, p in att.named_parameters():
        _close(p.grad, 2 * g1[n], 1e-6, n)
    _close(y.grad, 2 * dh1, 1e-6, "d h")
    att.zero_grad(set_to_none=True)
    assert all(p.grad is None for p in att.parameters())
    att.encoder_att.weight.requires_grad_(False)
    att.full_att.bias.requires_grad_(False)
    _loss(*att(x, y), gc, ga, "both").backward()
    for n, p in att.named_parameters():
        assert (p.grad is None) == (n in ("encoder_att.weight", "full_att.bias")), n
        if p.grad is not None:
            _close(p.grad, g1[n], 1e-6, n)


def test_only_h_skips_d_att1_and_its_gemms():
    att, enc, h, gc, ga = _module_case("fp32")
    for p in att.parameters():
        p.requires_grad_(False)
    counts = []
    for enc_grad in (False, True):
        x = enc.cuda().requires_grad_(enc_grad)
        y = h.cuda().requires_grad_(True)
        loss = _loss(*att(x, y), gc.cuda(), ga.cuda(), "both")
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        loss.backward()
        counts.append(_lib.launch_count() - n0)
        assert (x.grad is not None) == enc_grad and y.grad is not None
    # h only: s (d alpha term), the attention backward and d h = datt2 W_d.  d enc adds its GEMM and the alpha (x) dctx term
    assert counts[0] <= 3, counts
    assert counts[1] >= counts[0] + 2, counts


def test_double_backward_raises():
    att, enc, h, gc, ga = _module_case("fp32")
    y = h.cuda().requires_grad_(True)
    ctx, alpha = att(enc.cuda(), y)
    (gh,) = torch.autograd.grad((ctx * gc.cuda()).sum(), y, create_graph=True)
    with pytest.raises(RuntimeError):
        gh.sum().backward()


def test_stale_parameters_raise():
    att, enc, h, gc, ga = _module_case("fp32")
    ctx, alpha = att(enc.cuda(), h.cuda())
    with torch.no_grad():
        att.decoder_att.weight.mul_(1.0)
    with pytest.raises(_lib.LatexOcrB200Error):
        _loss(ctx, alpha, gc.cuda(), ga.cuda(), "both").backward()


def test_fused_train_step_after_autograd_use_of_decoder_attention():
    rm = _oracle()
    V = 40
    pe, pd = rm.init_params(V, seed=1)
    img, formula = rm.synthetic_batch(2, 32, 64, V, 3, 6, seed=2)
    m = build_model(V, pe, pd, "fp32")
    att = m.decoder.attention
    g = torch.Generator().manual_seed(9)
    enc = (torch.randn(3, 20, 512, generator=g) * 0.5).cuda().requires_grad_(True)
    h = torch.randn(3, 512, generator=g).cuda()
    m.decoder.zero_grad(set_to_none=True)
    ctx, alpha = att(enc, h)
    (ctx.sum() + (alpha ** 2).sum()).backward()
    for n, p in att.named_parameters():          # the gradients land in the decoder's p.grad
        assert p.grad is not None and dict(m.decoder.named_parameters())["attention." + n] is p, n
    assert enc.grad is not None
    m.train_step(img.cuda(), formula.cuda(), sync=True)
    for k, p in m.decoder.named_parameters():
        assert p.grad is not None and torch.equal(p.grad, grad_view(m.decoder.store, p)), k
    assert m.decoder.store.grad.abs().sum().item() > 0


def test_deterministic_backward_is_bit_reproducible():
    torch.manual_seed(11)
    att = Attention(512, 512, 512, precision="bf16")
    g = torch.Generator().manual_seed(12)
    enc = (torch.randn(8, 868, 512, generator=g) * 0.5).cuda()
    h = torch.randn(8, 512, generator=g).cuda()
    gc, ga = torch.randn(8, 512, generator=g).cuda(), torch.randn(8, 868, generator=g).cuda()
    with _lib.option(deterministic=1):
        runs = []
        for _ in range(2):
            att.zero_grad(set_to_none=True)
            x, y = enc.clone().requires_grad_(True), h.clone().requires_grad_(True)
            _loss(*att(x, y), gc, ga, "both").backward()
            runs.append([x.grad, y.grad] + [p.grad.clone() for p in att.parameters()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
