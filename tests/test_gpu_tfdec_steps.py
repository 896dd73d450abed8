"""-m gpu: the TensorFlow-flavour decoder's time loop (lo_tfdec_forward / lo_tfdec_backward, csrc/lo_tfdecoder.cuh) step by step
against float64, under the step schedules.

Each case runs tf_decoder.Decoder.run_forward (with the loss) and run_backward, then rebuilds every stored per-step quantity in
float64 (tests/tfdec_step_ref.py) from the operands the kernel of that step read: the values the workspace holds from the previous
launch (read through tfdec_step_ref.carve, the layout of tf_carve), rounded to bf16 where the kernel reads a bf16 mirror (xh_bf,
hd_bf, ctx_bf, dout2_bf, dz_bf, dlogits_bf on the tensor-core path), and the weights as the kernels see them (bf16 shadows in bf16,
the fp32 master otherwise; lstm.bias, att_beta and the initial-state biases fp32).  So an error never compounds across steps.

Bounds (element-wise; S = the float64 sum of the magnitudes of the terms of the exact value):
  * GEMMs and reductions (att_img, ptab, initpre, z + ptab, out2, o's products, logits, dologit, dctx, dh, every hoisted weight
    gradient, dptab, d enc):  |y - ref| <= 2^-16 S.  bf16 products are exact in fp32 (fp32 x fp32 ones inside an FMA), so the
    error is the sum of the n roundings of the fp32 updates.  Each is at most 2^-24 of the running partial sum, which is at most S,
    and their signs are random, so the total is about sqrt(n) 2^-24 S; that is <= 2^-16 S for n <= 2^16, which covers every sum
    here (the longest are the d att_img sweep and g att_img.kernel, n = B R = 55,552 at b64, and the hoisted gradients, n = T B).
    In practice the margin is far larger: the terms have random signs, so the partial sums stay near sqrt(k) of one term rather
    than S, and the error scales with them (the recorded ratios below are all <= 0.1).
    bf16 outputs (att_img, d att_img in bf16): half a bf16 ulp of ref on top.  The row means: (R + 1) 2^-24 sum_r |enc| / R.
  * Pointwise kernels propagate the allowance e of their input: sigmoid is 1/4-Lipschitz, tanh 1-Lipschitz, plus 2^-21 (expf /
    tanhf within 2 ulp, the add and the division).  c and h from the kernel's own gates and c: 2^-22 (|f c_prev| + |i g|) and
    2^-21 |h|.  o_t = tanh(oc + oh) keep: (2^-16 S_oc + 2^-21) |keep| + 2^-23 |o|.  The o backward: the GEMM allowance of the d o
    it reads times |keep (1 - o^2)|, plus 2^-21 of itself.  The cell backward carries dc in float64 beside the kernel's fp32 chain
    with its allowance E_dc, as tests/test_gpu_decoder_steps.py does.
  * Cross entropy from the stored logits: the rule of tests/test_gpu_decoder_steps.py ((V + 8) 2^-24 on the log-sum-exp, p times
    that plus 2^-24 |l - lse| + 2^-22 on a probability).
  * Attention, bf16 path: the score's tanh is tanh.approx.f32, which the PTX ISA specifies with a maximum relative error of 2^-11
    (the ISA's figure for the half-precision variants is 2^-10.987; the bound uses eps = 2^-10.98 >= both).  With post = tanh(pre)
    and pre = att_img + att_h rounded once (2^-24 |pre|):
        score error  d_r <= sum_a |beta_a| (eps |post_a| + 2^-23 |pre_a|) + 2^-16 sum_a |beta_a post_a|
        alpha_r      <= alpha_r (d_r + sum_r' alpha_r' d_r') + 2^-21 alpha_r           (first order of the softmax)
        ctx_c        <= sum_r e_alpha_r |enc_rc| + 2^-16 sum_r alpha_r |enc_rc|
    Its backward reads the kernel's own alpha, ctx and d ctx: de_r <= alpha_r 2^-16 (sum_c |dctx enc_rc| + sum_c |dctx ctx_c|) +
    2^-23 |de_r|; d att_h (from the kernel's own de) and the d beta partials use 1 - post^2 of the approximate post:
    |d(1 - post^2)| <= 2 eps post^2 + 2^-22 |pre|, and |d post| <= eps |post| + 2^-23 |pre|, each plus 2^-16 of the magnitudes.
    fp32 uses tanhf: the same formulas with eps = 2^-22 (2 ulp).
  * Exact: hd = h x keep_h bit for bit and its bf16 mirror RN(hd); o exactly 0 where keep_o is 0; the start state copied from
    sinit; zeros in d logits past each row's length and in the padding columns [V, ldl); a token fed once gets exactly its one dz
    row in dptab, a token never fed exactly 0; under sampling, fed[b][t] is the lowest-index argmax of the kernel's own logits row
    of step t where the injected coin u < p, and formula[b][t] otherwise.  In the generic backward (the autograd route: d logits
    and d alphas from the caller), d logits is the caller's, copied to time-major rows bit for bit, with zero padding columns.
  * Sampling with a temperature tau (Gumbel-max with injected uniforms u_v): where u < p, fed[b][t] maximises
    x_v = l_v / tau - log(-log u_v) of the kernel's own logits.  The kernel evaluates x_v in fp32 (a division and two logf, each
    within 1 ulp), so |x_v - x64_v| <= 2^-22 (|l_v / tau| + |log(-log u_v)| + 1) = e_v: the token fed must have x64 >= max - 2 max e,
    and must be the float64 argmax wherever the runner-up trails by more than that.
  * Generic backward: sreg[b,t] = sum_r alpha d alpha by the GEMM rule; de then reads d alpha and the kernel's sreg, which adds
    alpha_r 2^-16 (|d alpha_r| + |sreg|) to its bound.
  * The logits padding columns [V, ldl) are never written (the head GEMMs have N = V): they keep the sentinel.

The workspace (all but the attention ticket counters and the buffers the backward zeroes itself: dxh, dc, dbeta_acc), logits,
alphas, the gradient store and d enc are filled with a finite sentinel before the call; it must not reach any checked quantity.
Under "deterministic" two runs from the same state must agree bit for bit in every output, stored buffer and gradient.

Worst |y - ref| / bound per quantity, over every case and schedule, measured on an H100 80GB HBM3 (700 W power limit); the whole
file (37 runs) ran in 14 s there:
    bf16 roundings (a value next to a rounding midpoint nears half an ulp): att_img 0.983, datt_img 0.996
    pointwise and cross entropy: c 0.469, h 0.446, dlogits 0.723, dpre_o 0.438, sinit 0.162, dinit 0.054, gates 0.026, o 0.016,
        dz 0.012, row loss 0.020, loss 0.007
    attention (tanh.approx rule): alphas 0.002, ctx 0.001, de 0.003, d att_h 0.012, d beta partials 0.011
    GEMMs and reductions (2^-16 S): att_img 0.983 (its bf16 rounding, above), ptab 0.013, mean 0.067, initpre 0.018, out2 0.015,
        logits 0.018, dologit 0.090, dctx 0.012, sreg 0.004, dptab 0.015, g lstm.kernel 0.033 / 0.021, g lstm.bias 0.011,
        g embedding 0.011, g att_h.kernel 0.016, g o_W_h 0.015, g o_W_c 0.016, g y_W_o 0.081, g att_beta 0.008,
        g att_img.kernel 0.035, g W_init 0.021, g b_init 0.011, d enc 0.028
"""
import pytest
import torch

import tfdec_step_ref as tr

pytestmark = pytest.mark.gpu

_SENTINEL = -1536.0
_ACC = 2.0 ** -16
_ULPS = 2.0 ** -21
_V = 500

# name: (precision, impl, B, R, T, (A, C), D, O, E, mode)  mode: None, "keep" (injected keep masks with zeros), "ss" (sampling
# with p = 0.5 and injected coins), "ssg" (ss with a temperature and injected Gumbel uniforms), "generic" (the autograd route's
# backward: d logits and d alphas from the caller).  t8: ragged lengths.  b64: the tools/tf_bench.py shape.  b72: wgmma step GEMMs
# (M > 64), split-K atomics in the backward, and B (T - 1) = 288 > 256 tokens for the ordered d ptab gather's scan.  a*: the A = C
# tanh instantiations.  d640: other K slices, a K[E:] offset of 64 and 4D = 2560 gate columns (a partial column block of the d ptab
# gather).
_CASES = {
    "t8": ("bf16", "tc", 8, 44, 7, (256, 512), 512, 512, 80, None),
    "b64": ("bf16", "tc", 64, 868, 3, (256, 512), 512, 512, 80, None),
    "b72": ("bf16", "tc", 72, 101, 5, (256, 512), 512, 512, 80, None),
    "a256": ("bf16", "tc", 8, 44, 4, (256, 256), 512, 512, 80, None),
    "a512": ("bf16", "tc", 6, 44, 4, (512, 512), 512, 512, 80, None),
    "a1024": ("bf16", "tc", 4, 30, 3, (1024, 1024), 512, 512, 80, None),
    "d640": ("bf16", "tc", 8, 44, 4, (256, 512), 640, 384, 64, None),
    "keep": ("bf16", "tc", 8, 44, 5, (256, 512), 512, 512, 80, "keep"),
    "ss": ("bf16", "tc", 8, 44, 6, (256, 512), 512, 512, 80, "ss"),
    "ssg": ("bf16", "tc", 8, 44, 6, (256, 512), 512, 512, 80, "ssg"),
    "generic": ("bf16", "tc", 8, 44, 5, (256, 512), 512, 512, 80, "generic"),
    "fp32": ("fp32", "simt", 8, 44, 5, (256, 512), 512, 512, 80, "keep"),
    "bf16simt": ("bf16", "simt", 8, 44, 5, (256, 512), 512, 512, 80, None),
}

_SCHEDULES = {
    "default": ({}, list(_CASES)),
    "deterministic": ({"deterministic": 1}, ["t8", "b64", "b72", "d640", "keep", "ss", "generic"]),
    "skinny_mma0": ({"skinny_mma": 0}, ["t8", "b64"]),
    "skinny_tma0": ({"skinny_tma": 0}, ["t8"]),
    "skinny8_0": ({"skinny8": 0}, ["b72"]),
    "wgrad256": ({"wgrad256": 1}, ["b64", "b72"]),
    "pdl0": ({"pdl": 0}, ["t8", "b72"]),
    "att_cluster0": ({"att_cluster": 0}, ["b64", "b72"]),
    "att_cluster2": ({"att_cluster": 2}, ["b64"]),
    "att_nsplit3": ({"att_nsplit": 3}, ["t8", "a1024"]),
    "att_l2_keep0": ({"att_l2_keep_mb": 0}, ["b64"]),
    "conv_mc0": ({"conv_mc": 0}, ["t8", "b72"]),
}
_PARAMS = [(s, c) for s, (_, cs) in _SCHEDULES.items() for c in cs]
_WORST = {}
# the backward zeroes these itself, and the attention ticket counters must start at zero
_NOT_FILLED = ("attwork", "dxh", "dc", "dbeta_acc")


def _rn(x):
    return x.bfloat16().double()


def _half_ulp_bf16(ref):
    _, e = torch.frexp(ref)
    return torch.where(ref != 0, torch.ldexp(torch.full_like(ref, 0.5), e - 8), torch.zeros_like(ref))


class _Checker:
    def __init__(self, tag):
        self.tag = tag
        self.worst = {}

    def bound(self, name, y, ref, bound):
        d = (y.double() - ref).abs()
        bound = torch.broadcast_to(torch.as_tensor(bound, dtype=torch.float64, device=d.device), d.shape)
        ok = d <= bound
        if not bool(ok.all()):
            bad = (~ok).nonzero()
            i = tuple(bad[0].tolist())
            raise AssertionError("%s %s: %d of %d elements outside the bound; first at %s: got %r, float64 %r, bound %.3g"
                                 % (self.tag, name, bad.shape[0], y.numel(), i, y[i].item(), ref[i].item(), bound[i].item()))
        r = torch.where(bound > 0, d / bound.clamp_min(1e-300), torch.zeros_like(d)).max().item() if d.numel() else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)

    def gemm(self, name, y, ref, S):
        self.bound(name, y, ref, _ACC * S + 1e-38)

    def exact(self, name, y, ref):
        assert torch.equal(y, ref.to(y.dtype)), "%s %s: not bit for bit" % (self.tag, name)

    def value(self, name, y, v):
        assert bool((y == v).all()), "%s %s: expected every element to be %r" % (self.tag, name, v)


def _model(case, seed):
    from latex_ocr_b200.tf_decoder import Decoder
    from util import Cfg
    precision, impl, B, R, T, (A, C), D, O, E, mode = _CASES[case]
    torch.manual_seed(seed)
    cfg = Cfg(attn_cell_config={"num_units": D, "dim_e": A, "dim_o": O, "dim_embeddings": E}, max_length_formula=10)
    dec = Decoder(cfg, _V, _V - 1, device="cuda", precision=precision, impl=impl, channels=C)
    with torch.no_grad():
        dec.lstm.bias.uniform_(-0.3, 0.3)        # zero at init: give the bias path something to add
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    enc = torch.randn(B, R, C, device="cuda", generator=g).to(dec.tdtype)
    formula = torch.randint(0, _V, (B, T), device="cuda", generator=g)
    formula[1] = formula[0]                      # repeated tokens: rows of dptab that sum several dz rows
    formula[0, 1] = formula[0, 0]
    lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(seed + 2))
    lengths[0] = T
    keep_h = keep_o = None
    if mode == "keep":
        keep_h = (torch.rand(B, T, D, device="cuda", generator=g) >= 0.3).float() / 0.7
        keep_o = (torch.rand(B, T, O, device="cuda", generator=g) >= 0.3).float() / 0.7
    dl = dal = None
    if mode in ("ss", "ssg"):
        dec._ss_u = torch.rand(B, T, device="cuda", generator=g)
    if mode == "ssg":
        dec._ss_gu = torch.rand(B, T, _V, device="cuda", generator=g).clamp_min(1e-6)
    if mode == "generic":
        dl = 1e-3 * torch.randn(B, T, _V, device="cuda", generator=g)
        dal = 1e-2 * torch.randn(B, T, R, device="cuda", generator=g)
    return dict(dec=dec, enc=enc, formula=formula, lengths=lengths, keep_h=keep_h, keep_o=keep_o, mode=mode,
                tau=0.7 if mode == "ssg" else None, dl=dl, dal=dal)


def _run(c):
    """One forward + backward from sentinel-filled buffers; returns (ws, views of ws["ws"]).  Generic mode: the forward without
    the loss, then the backward of the autograd route (Decoder._backward_impl) with the case's d logits and d alphas."""
    dec, enc, formula, keep_h, keep_o = c["dec"], c["enc"], c["formula"], c["keep_h"], c["keep_o"]
    B, R, C = enc.shape
    T = formula.shape[1]
    ssp, tau = dec.sampling_scalars(0.5, c["tau"] or 0.0) if c["mode"] in ("ss", "ssg") else (None, None)
    generic = c["mode"] == "generic"
    lengths = None if generic else c["lengths"]
    ws = dec.run_forward(enc, formula, lengths, keep_h, keep_o, ss_prob=ssp, ss_temp=tau)     # allocates the workspace
    torch.cuda.synchronize()
    layout, _ = tr.carve(B, T, R, C, dec.A, dec.D, dec.O, dec.E, dec.V, ws["ldl"], dec.precision == "bf16")
    v = tr.views_of(ws["ws"], layout)
    for k, t in v.items():
        if k not in _NOT_FILLED and t.is_floating_point():
            t.fill_(_SENTINEL)
    for k in ("logits", "alphas", "denc"):
        ws[k].fill_(_SENTINEL)
    dec.store.grad.fill_(_SENTINEL)
    ws = dec.run_forward(enc, formula, lengths, keep_h, keep_o, ss_prob=ssp, ss_temp=tau)
    if generic:
        dec._backward_impl({"ws": ws, "args": ws["args"], "shape": tuple(enc.shape), "dtype": enc.dtype}, c["dl"], c["dal"], None)
    else:
        dec.run_backward(ws)
    torch.cuda.synchronize()
    return ws, v


def _params(dec):
    """TF-layout float64 weights as the kernels see them."""
    S = dec.store
    p = {}
    for n in ("att_img.kernel", "att_h.kernel", "o_W_h", "lstm.kernel", "o_W_c", "y_W_o", "W_c_0", "W_h_0", "W_o_0"):
        p[n] = S.w(n).double().t()
    for n in ("embedding_table", "start_token"):
        p[n] = S.w(n).double()
    for n in ("att_beta", "lstm.bias", "b_c_0", "b_h_0", "b_o_0"):
        p[n] = S.f32(n).double()
    return p


def _att_eps(dec):
    return 2.0 ** -10.98 if dec.precision == "bf16" else 2.0 ** -22


def _check(ck, c, ws, v):
    dec, enc, formula, lengths, keep_h, keep_o = c["dec"], c["enc"], c["formula"], c["lengths"], c["keep_h"], c["keep_o"]
    ss = c["mode"] in ("ss", "ssg")
    generic = c["mode"] == "generic"
    S = dec.store
    B, R, C = enc.shape
    T = formula.shape[1]
    A, D, O, E, V = dec.A, dec.D, dec.O, dec.E, dec.V
    G, XH = 4 * D, O + D
    tc = dec.impl == "tc" and dec.precision == "bf16"
    act = _rn if tc else (lambda x: x.double())
    eps = _att_eps(dec)
    p = _params(dec)
    beta = p["att_beta"]
    encd = enc.double()
    KE = p["lstm.kernel"][E:]                                        # [O+D][4D]
    kh = None if keep_h is None else keep_h.transpose(0, 1).double()       # [T][B][D]
    ko = None if keep_o is None else keep_o.transpose(0, 1).double()

    # ---- prologue: att_img, ptab, the row means, the initial state
    att_img = v["att_img"]
    ref, Sa = tr.linear(encd, p["att_img.kernel"])
    ck.bound("att_img", att_img, ref, _ACC * Sa + (_half_ulp_bf16(ref) if att_img.dtype == torch.bfloat16 else 0))
    emb = torch.cat([p["embedding_table"], p["start_token"][None]], 0)
    ref, Sp = tr.linear(emb, p["lstm.kernel"][:E], p["lstm.bias"])
    ck.gemm("ptab", v["ptab"], ref, Sp)
    ck.bound("mean", v["mean"], encd.mean(1), (R + 1) * 2.0 ** -24 * encd.abs().mean(1))
    mean = v["mean"].double()
    wi, bi = tr.w_init(p)
    ref, Si = tr.linear(mean, wi, bi)
    ck.gemm("initpre", v["initpre"], ref, Si)
    ck.bound("sinit", v["sinit"], torch.tanh(v["initpre"].double()), _ULPS)
    s0 = v["sinit"]
    ck.exact("c0", v["call"][0], s0[:, :D])
    ck.exact("xh0 h", v["xh"][0][:, O:], s0[:, D:2 * D])
    ck.exact("xh0 o", v["xh"][0][:, :O], s0[:, 2 * D:])

    # ---- the forward time loop from the kernel's own inputs
    fed = ws["fed"] if ss else None
    tok = tr.tokens_consumed(formula, V, fed)                       # [B][T]
    ptab = v["ptab"].double()
    aimg = att_img.double()
    lg_all = ws["logits"]
    for t in range(T):
        xh = v["xh"][t]
        z, Sz = tr.linear(act(xh), KE)
        pt = ptab[tok[:, t]]
        pre = z + pt
        e_pre = _ACC * (Sz + pt.abs())
        gts = v["gates"][t]
        for q, (fn, lip, sh) in enumerate(((torch.sigmoid, 0.25, 0.0), (torch.tanh, 1.0, 0.0), (torch.sigmoid, 0.25, 1.0),
                                           (torch.sigmoid, 0.25, 0.0))):
            sl = slice(q * D, (q + 1) * D)
            ck.bound("gates", gts[:, sl], fn(pre[:, sl] + sh), lip * e_pre[:, sl] + _ULPS)
        i, g, f, o = gts.double().chunk(4, 1)
        cp = v["call"][t].double()
        ck.bound("c", v["call"][t + 1], f * cp + i * g, 2.0 ** -22 * ((f * cp).abs() + (i * g).abs()) + 1e-38)
        href = o * torch.tanh(v["call"][t + 1].double())
        h = v["xh"][t + 1][:, O:]
        ck.bound("h", h, href, 2.0 ** -21 * href.abs() + 1e-38)
        if keep_h is not None:
            ck.exact("hd", v["hd"][t], h * keep_h[:, t])
            if tc:
                ck.exact("hd_bf", v["hd_bf"][t], v["hd"][t].bfloat16())
            hsrc = v["hd"][t]
        else:
            hsrc = h
        if tc:
            ck.exact("xh_bf", v["xh_bf"][t + 1], v["xh"][t + 1].bfloat16())
        ref, S2 = tr.linear(act(hsrc), tr.w_cat2(p))
        ck.gemm("out2", v["out2"][t], ref, S2)
        # attention from the kernel's own att_img and att_h
        att_h = v["out2"][t][:, :A].double()
        pre_a = aimg + att_h[:, None, :]
        post = torch.tanh(pre_a)
        e_sc = (post * beta).sum(-1)
        d_r = ((eps * post.abs() + 2.0 ** -23 * pre_a.abs()) * beta.abs()).sum(-1) + _ACC * (post * beta).abs().sum(-1)
        alpha = torch.softmax(e_sc, 1)
        e_al = alpha * (d_r + (alpha * d_r).sum(1, keepdim=True)) + _ULPS * alpha
        ck.bound("alphas", ws["alphas"][:, t], alpha, e_al + 1e-38)
        ctx = torch.einsum("br,brc->bc", alpha, encd)
        e_ctx = torch.einsum("br,brc->bc", e_al, encd.abs()) + _ACC * torch.einsum("br,brc->bc", alpha, encd.abs())
        ck.bound("ctx", v["ctx"][t], ctx, e_ctx + 1e-38)
        if tc:
            ck.exact("ctx_bf", v["ctx_bf"][t], v["ctx"][t].bfloat16())
        oc, Soc = tr.linear(act(v["ctx"][t]), p["o_W_c"])
        oref = torch.tanh(oc + v["out2"][t][:, A:].double())
        kt = torch.ones_like(oref) if ko is None else ko[t]
        ck.bound("o", v["xh"][t + 1][:, :O], oref * kt, (_ACC * Soc + _ULPS) * kt.abs() + 2.0 ** -23 * (oref * kt).abs() + 1e-38)
        if ko is not None:
            ck.value("o where keep_o is 0", v["xh"][t + 1][:, :O][ko[t] == 0], 0.0)
        # head
        ref, Sl = tr.linear(act(v["xh"][t + 1][:, :O]), p["y_W_o"])
        ck.gemm("logits", lg_all[t][:, :V], ref, Sl)
        if ss:
            u = dec._ss_u[:, t]
            if c["tau"] is None:
                am = lg_all[t][:, :V].argmax(-1)
                want = torch.where(u < 0.5, am, formula[:, t])
                assert torch.equal(fed[:, t], want), "%s fed[:, %d]: %s, want %s" % (ck.tag, t, fed[:, t].tolist(), want.tolist())
            else:
                lt = lg_all[t][:, :V].double() / c["tau"]
                gm = -torch.log(-torch.log(dec._ss_gu[:, t].double()))
                x = lt + gm
                tol = 2 * (2.0 ** -22 * (lt.abs() + gm.abs() + 1)).max(-1).values
                top2 = x.topk(2, -1)
                sampled = u < 0.5
                assert torch.equal(fed[:, t][~sampled], formula[:, t][~sampled]), "%s fed[:, %d] where u >= p" % (ck.tag, t)
                xf = x.gather(-1, fed[:, t][:, None])[:, 0]
                assert bool((xf[sampled] >= top2.values[sampled, 0] - tol[sampled]).all()), "%s fed[:, %d]: not a Gumbel max" % (ck.tag, t)
                clear = sampled & (top2.values[:, 0] - top2.values[:, 1] > tol)
                assert torch.equal(fed[:, t][clear], top2.indices[clear, 0]), "%s fed[:, %d]: not the Gumbel argmax" % (ck.tag, t)
    ck.value("logits padding columns (never written)", lg_all[:, :, V:], _SENTINEL)

    # ---- cross entropy, or the caller's d logits (generic)
    if generic:
        ck.exact("dlogits (generic, time-major)", v["dlogits"][:, :, :V], c["dl"].transpose(0, 1))
        ck.value("dlogits padding columns", v["dlogits"][:, :, V:], 0.0)
        if tc:
            ck.exact("dlogits_bf", v["dlogits_bf"], v["dlogits"].bfloat16())
        al_ = ws["alphas"].double()
        dal = c["dal"].double()
        ck.gemm("sreg", v["sreg"], (al_ * dal).sum(-1), (al_ * dal).abs().sum(-1))
    else:
        _check_ce(ck, c, ws, v, tc)
    _check_backward(ck, c, ws, v, p, act, eps, tok, generic)


def _check_ce(ck, c, ws, v, tc):
    formula, lengths = c["formula"], c["lengths"]
    T, B = formula.shape[1], formula.shape[0]
    V = c["dec"].V
    lg_all = ws["logits"]
    valid = (torch.arange(T)[:, None] < lengths[None, :]).cuda()     # [T][B]
    nvalid = int(valid.sum())
    inv_n = 1.0 / nvalid
    lg = lg_all[:, :, :V].double()[valid]
    tg = formula.t()[valid]
    row, dl = tr.cross_entropy(lg, tg, inv_n)
    lse = torch.logsumexp(lg, -1)
    d_lse = (V + 8) * 2.0 ** -24 + 2.0 ** -23 * lse.abs()
    pr = torch.exp(lg - lse[:, None])
    d_p = pr * (d_lse[:, None] + 2.0 ** -24 * (lg - lse[:, None]).abs() + 2.0 ** -22)
    row_b = d_lse + 2.0 ** -23 * (lse.abs() + lg.gather(-1, tg[:, None])[:, 0].abs())
    ck.bound("row_loss", v["row_loss"][valid], row, row_b)
    ck.value("row_loss past the length", v["row_loss"][~valid], 0.0)
    ck.bound("dlogits", v["dlogits"][:, :, :V][valid], dl, d_p * inv_n + 2.0 ** -23 * dl.abs())
    ck.value("dlogits past the length", v["dlogits"][~valid], 0.0)
    ck.value("dlogits padding columns", v["dlogits"][:, :, V:], 0.0)
    if tc:
        ck.exact("dlogits_bf", v["dlogits_bf"], v["dlogits"].bfloat16())
    ck.bound("loss", ws["loss"][0:1], (row.sum() * inv_n).reshape(1), (inv_n * row_b.sum() + _ACC * inv_n * row.abs().sum()).reshape(1))


def _check_backward(ck, c, ws, v, p, act, eps, tok, generic):
    dec, enc, formula, keep_h, keep_o = c["dec"], c["enc"], c["formula"], c["keep_h"], c["keep_o"]
    S = dec.store
    B, R, C = enc.shape
    T = formula.shape[1]
    A, D, O, E, V = dec.A, dec.D, dec.O, dec.E, dec.V
    G, XH = 4 * D, O + D
    tc = dec.impl == "tc" and dec.precision == "bf16"
    beta = p["att_beta"]
    encd = enc.double()
    KE = p["lstm.kernel"][E:]
    kh = None if keep_h is None else keep_h.transpose(0, 1).double()
    ko = None if keep_o is None else keep_o.transpose(0, 1).double()
    aimg = v["att_img"].double()
    s0 = v["sinit"]
    mean = v["mean"].double()
    wi, _ = tr.w_init(p)
    emb = torch.cat([p["embedding_table"], p["start_token"][None]], 0)
    dalk = c["dal"].double() if generic else None
    sregk = v["sreg"].double() if generic else None

    # ---- backward: d o from the logits, then the loop in reverse from the kernel's own stored values
    WY = p["y_W_o"].t()                                                # [V][O]
    x = act(v["dlogits"][:, :, :V])
    ck.gemm("dologit", v["dologit"], x @ WY, x.abs() @ WY.abs())
    dc = torch.zeros(B, D, dtype=torch.float64, device="cuda")
    e_dc = torch.zeros_like(dc)
    W4 = torch.cat([p["att_h.kernel"].t(), p["o_W_h"].t()], 0)         # [A+O][D]: d hd = dout2 @ W4
    dbeta = torch.zeros(B, A, dtype=torch.float64, device="cuda")
    e_dbeta = torch.zeros_like(dbeta)
    for t in range(T - 1, -1, -1):
        if t + 1 < T:
            xz = act(v["dz"][t + 1])
            dxh_, e_dxh = xz @ KE.t(), _ACC * (xz.abs() @ KE.abs().t())
        else:
            dxh_ = torch.zeros(B, XH, dtype=torch.float64, device="cuda")
            e_dxh = torch.zeros_like(dxh_)
        dvo = dxh_[:, :O] + v["dologit"][t].double()
        e_dvo = e_dxh[:, :O] + 2.0 ** -24 * dvo.abs()
        o_st = v["xh"][t + 1][:, :O].double()
        dpre = tr.o_backward(dxh_[:, :O], v["dologit"][t].double(), None if ko is None else ko[t], o_st)
        kt = torch.ones_like(o_st) if ko is None else ko[t]
        ou = torch.where(kt != 0, o_st / torch.where(kt != 0, kt, torch.ones_like(kt)), torch.zeros_like(o_st))
        ck.bound("dpre_o", v["dout2"][t][:, A:], dpre, e_dvo * (kt * (1 - ou * ou)).abs() + _ULPS * dpre.abs() + 1e-38)
        if tc:
            ck.exact("dout2_bf", v["dout2_bf"][t], v["dout2"][t].bfloat16())
        xo = act(v["dout2"][t][:, A:])
        ck.gemm("dctx", v["dctx"][t], xo @ p["o_W_c"].t(), xo.abs() @ p["o_W_c"].abs().t())
        # attention backward from the kernel's own alpha, ctx, d ctx and de
        al = ws["alphas"][:, t].double()
        ctxk = v["ctx"][t].double()
        dctx = v["dctx"][t].double()
        att_h = v["out2"][t][:, :A].double()
        if generic:
            de, _, _ = tr.attention_backward(aimg, encd, att_h, beta, al, ctxk, dctx, dalk[:, t], sregk[:, t])
        else:
            de, _, _ = tr.attention_backward(aimg, encd, att_h, beta, al, ctxk, dctx)
        e_de = (al * _ACC * (torch.einsum("bc,brc->br", dctx.abs(), encd.abs()) + (dctx * ctxk).abs().sum(-1, keepdim=True))
                + 2.0 ** -23 * de.abs())
        if generic:
            e_de = e_de + al * _ACC * (dalk[:, t].abs() + sregk[:, t, None].abs())
        ck.bound("de", v["de"][:, t], de, e_de + 1e-38)
        dek = v["de"][:, t].double()
        pre_a = aimg + att_h[:, None, :]
        post = torch.tanh(pre_a)
        dact = 1 - post * post
        e_dact = 2 * eps * post * post + 2.0 ** -22 * pre_a.abs()
        datt_h = torch.einsum("br,bra->ba", dek, dact) * beta
        e_datt = (torch.einsum("br,bra->ba", dek.abs(), e_dact) + _ACC * torch.einsum("br,bra->ba", dek.abs(), dact)) * beta.abs()
        ck.bound("d att_h", v["dout2"][t][:, :A], datt_h, e_datt + 2.0 ** -23 * datt_h.abs() + 1e-38)
        dbeta += torch.einsum("br,bra->ba", dek, post)
        e_dbeta += (torch.einsum("br,bra->ba", dek.abs(), eps * post.abs() + 2.0 ** -23 * pre_a.abs())
                    + _ACC * torch.einsum("br,bra->ba", dek.abs(), post.abs()))
        # the cell backward: dh = recurrent part + keep (d hd)
        xd = act(v["dout2"][t])
        dhd, e_dhd = xd @ W4, _ACC * (xd.abs() @ W4.abs())
        khd = torch.ones_like(dhd) if kh is None else kh[t]
        dh = dxh_[:, O:] + khd * dhd
        e_dh = e_dxh[:, O:] + e_dhd * khd.abs() + 2.0 ** -23 * dh.abs()
        gts = v["gates"][t].double()
        i, g, f, o = gts.chunk(4, 1)
        cc = v["call"][t + 1].double()
        cp = v["call"][t].double()
        th = torch.tanh(cc)
        dz, dct, dcp = tr.lstm_backward(dh, torch.zeros_like(dh), None, dc, gts, cp, cc)
        e_dct = (e_dc + e_dh * (o * (1 - th * th)).abs() + (dh * o).abs() * (2 * th.abs() * 2.0 ** -22 * th.abs() + 2.0 ** -23)
                 + 2.0 ** -22 * (dc.abs() + (dh * o * (1 - th * th)).abs()))
        bnd = torch.cat([e_dct * (g * i * (1 - i)).abs(), e_dct * (i * (1 - g * g)).abs() + (dct * i).abs() * 2.0 ** -23,
                         e_dct * (cp * f * (1 - f)).abs(),
                         e_dh * (th * o * (1 - o)).abs() + (dh * o * (1 - o)).abs() * 2.0 ** -22 * th.abs()], 1) + _ULPS * dz.abs()
        ck.bound("dz", v["dz"][t], dz, bnd + 1e-38)
        if tc:
            ck.exact("dz_bf", v["dz_bf"][t], v["dz"][t].bfloat16())
        dc, e_dc = dcp, e_dct * f.abs() + 2.0 ** -24 * dcp.abs()
    ck.bound("dbeta partials", v["dbeta_acc"], dbeta, e_dbeta + 2.0 ** -24 * T * dbeta.abs() + 1e-38)
    xz = act(v["dz"][0])
    dx0, e_dx0 = xz @ KE.t(), _ACC * (xz.abs() @ KE.abs().t())
    s0d = s0.double()
    ds = torch.cat([dc, dx0[:, O:], dx0[:, :O]], 1)
    e_ds = torch.cat([e_dc, e_dx0[:, O:], e_dx0[:, :O]], 1)
    dinit = tr.initial_backward(ds, s0d)
    ck.bound("dinit", v["dinit"], dinit, e_ds * (1 - s0d * s0d) + _ULPS * dinit.abs() + 1e-38)

    # ---- hoisted gradients from the stored per-step values
    def tn(name, y, X, Y):
        ck.gemm(name, y, X.t() @ Y, X.abs().t() @ Y.abs())

    def colsum(name, y, X):
        ck.gemm(name, y, X.double().sum(0), X.double().abs().sum(0))

    TB = T * B
    XHr = v["xh"][:T].reshape(TB, XH)
    DZ = v["dz"].reshape(TB, G)
    tn("g lstm.kernel [o; h]", S.g("lstm.kernel")[:, E:].t(), act(XHr), act(DZ))
    toks = tok.t().reshape(-1)
    hit = (toks[:, None] == torch.arange(V + 1, device="cuda")[None, :]).double()
    tn("dptab", v["dptab"], hit, DZ.double())
    cnt = hit.sum(0)
    ck.value("dptab of tokens never fed", v["dptab"][cnt == 0], 0.0)
    once = (cnt == 1).nonzero()[:, 0]
    if len(once):
        src = hit[:, once].argmax(0)
        ck.exact("dptab of tokens fed once", v["dptab"][once], DZ[src])
    dpt = v["dptab"].double()
    ge = S.g("embedding_table").double()
    gst = S.g("start_token").double()
    KEm = p["lstm.kernel"][:E]
    ck.gemm("g embedding_table | start_token", torch.cat([ge, gst[None]], 0), dpt @ KEm.t(), dpt.abs() @ KEm.abs().t())
    tn("g lstm.kernel [emb]", S.g("lstm.kernel")[:, :E].t(), emb, dpt)
    colsum("g lstm.bias", S.g("lstm.bias"), v["dptab"])
    Hs = v["hd"] if keep_h is not None else v["xh"][1:, :, O:]
    H = act(Hs.reshape(TB, D))
    DO2 = v["dout2"].reshape(TB, A + O)
    tn("g att_h.kernel", S.g("att_h.kernel").t(), H, act(DO2[:, :A]))
    tn("g o_W_h", S.g("o_W_h").t(), H, act(DO2[:, A:]))
    tn("g o_W_c", S.g("o_W_c").t(), act(v["ctx"].reshape(TB, C)), act(DO2[:, A:]))
    tn("g y_W_o", S.g("y_W_o").t(), act(v["xh"][1:, :, :O].reshape(TB, O)), act(v["dlogits"][:, :, :V].reshape(TB, V)))
    colsum("g att_beta", S.g("att_beta"), v["dbeta_acc"])
    # d att_img: one sweep over t from the kernel's own de and att_h
    deall = v["de"].double()                                           # [B][T][R]
    da = torch.zeros(B, R, A, dtype=torch.float64, device="cuda")
    e_da = torch.zeros_like(da)
    for t in range(T):
        pre_a = aimg + v["out2"][t][:, None, :A].double()
        post = torch.tanh(pre_a)
        da += deall[:, t, :, None] * (1 - post * post)
        e_da += deall[:, t, :, None].abs() * (_ACC * (1 - post * post) + 2 * eps * post * post + 2.0 ** -22 * pre_a.abs())
    da, e_da = da * beta, e_da * beta.abs()
    datt = v["datt_img"]
    ck.bound("datt_img", datt, da, e_da + 2.0 ** -23 * da.abs() + (_half_ulp_bf16(da) if datt.dtype == torch.bfloat16 else 0) + 1e-38)
    d1 = datt.double().reshape(B * R, A)
    tn("g att_img.kernel", S.g("att_img.kernel").t(), encd.reshape(B * R, C), d1)
    dinitk = v["dinit"].double()
    gw = torch.cat([S.g("W_c_0"), S.g("W_h_0"), S.g("W_o_0")], 0).t()
    tn("g W_init", gw, mean, dinitk)
    colsum("g b_init", torch.cat([S.g("b_c_0"), S.g("b_h_0"), S.g("b_o_0")]), v["dinit"])
    Wimg = p["att_img.kernel"]                                         # [C][A]
    al = ws["alphas"].double()
    dcx = v["dctx"].transpose(0, 1).double()                           # [B][T][C]
    ref = ((d1 @ Wimg.t()).view(B, R, C) + torch.einsum("btr,btc->brc", al, dcx) + (dinitk @ wi.t() / R)[:, None, :])
    Sref = ((d1.abs() @ Wimg.abs().t()).view(B, R, C) + torch.einsum("btr,btc->brc", al.abs(), dcx.abs())
            + (dinitk.abs() @ wi.abs().t() / R)[:, None, :])
    ck.gemm("d enc", ws["denc"], ref, Sref)
    ck.value("no sentinel in the gradients", (S.grad == _SENTINEL).any().reshape(1), False)


def _outputs(dec, ws):
    return [ws[k].clone() for k in ("ws", "logits", "alphas", "loss", "denc")] + [dec.store.grad.clone()] + (
        [ws["fed"].clone()] if ws.get("fed") is not None else [])


@pytest.mark.parametrize("schedule,case", _PARAMS, ids=["%s-%s" % sc for sc in _PARAMS])
def test_tfdec_steps_vs_float64(schedule, case):
    """Every stored per-step quantity of the forward and backward time loops, the hoisted gradients and d enc within the bounds of
    the module docstring of float64 from the kernel's own operands.  Under "deterministic" two runs from the same state must agree
    bit for bit."""
    from latex_ocr_b200 import _lib
    opts, _ = _SCHEDULES[schedule]
    seed = sorted(_CASES).index(case)
    c = _model(case, seed)
    dec = c["dec"]
    with _lib.option(**opts):
        ws, v = _run(c)
        first = _outputs(dec, ws) if "deterministic" in opts else None
        ck = _Checker("%s %s" % (schedule, case))
        _check(ck, c, ws, v)
        if first is not None:
            ws, _ = _run(c)
            names = ["ws", "logits", "alphas", "loss", "denc", "grad", "fed"]
            for n, a, b in zip(names, first, _outputs(dec, ws)):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "deterministic: two runs differ in " + n
    for k, r in ck.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), r)
    print("\n%-24s %s" % (ck.tag, "  ".join("%s %.3f" % kv for kv in sorted(ck.worst.items()))))


def test_zz_worst_ratios():
    """Prints the worst |y - ref| / bound per quantity over the cases above (run after them)."""
    if not _WORST:
        pytest.skip("run with the step tests")
    print("\nworst |y - ref| / bound per quantity:")
    for k, r in sorted(_WORST.items()):
        print("  %-36s %.4f" % (k, r))
