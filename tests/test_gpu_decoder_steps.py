"""-m gpu: the decoder's time loop (lo_decoder_forward / lo_decoder_backward, csrc/lo_decoder.cu) step by step against float64,
under every step schedule.

Each case runs DecoderWithAttention.run_forward(..., need_grad=True) and run_backward, then rebuilds every stored per-step
quantity in float64 (tests/decoder_step_ref.py) from the operands the kernel of that step read: the values the workspace holds
from the previous launch, rounded to bf16 where the kernel reads a bf16 mirror (RN_bf16(hall), RN_bf16(gctx), RN_bf16(hd),
RN_bf16(dcat), RN_bf16(dlogits), RN_bf16(dptab), RN_bf16(alphas), RN_bf16(dctx) on the tensor-core path), and the weights as
the kernels see them (bf16 shadows in bf16, the fp32 master otherwise; biases and full_att.weight fp32).  So an error never
compounds across steps: each check sees one launch's arithmetic.

The two-layer decoder of the extension (cases b8l2, b72maskl2) runs the phases the way TwoLayerDecoder drives them, with
snapshots between them: the phase-1 forward must leave the logits and row_loss holding the sentinel and write hd = hall x
multiplier; DecoderLayer2 over hd is checked launch by launch with tests/test_gpu_lstmseq_steps.py's checks on its own
workspace; the phase-2 forward's logits are fc(RN_bf16(h2)) and its cross entropy is checked as in phase 0; the phase-2 backward
writes dhd = dlogits W_fc and the fc gradients and leaves every other gradient holding the sentinel; the phase-1 backward's
time loop takes dh = (layer 2's d x, read from dhd) x multiplier + carried.  Checks and bounds are the ones of phase 0 (helpers
shared through tests/step_check.py).

Bounds (every check, element-wise; S = the float64 sum of the magnitudes of the terms of the exact value):
  * fp32 GEMM / reduction outputs (out1's att2 and hh blocks, ptab, logits, dhd, the dh and d gctx products, every hoisted
    weight gradient, d encoder_out):  |y - ref| <= 2^-16 S.  bf16 products are exact in fp32 (and fp32 x fp32 products are
    exact inside an FMA); each of the n <= 2^12 fp32 updates of a sum errs by at most 2^-24 of a running sum bounded by S, with
    random sign, so about sqrt(n) 2^-24 S <= 2^-18 S; 2^-16 S leaves a factor of four and is still far below one lost term.
  * h0, c0 on the tensor-core path: the fp32 row means enter as hi + lo bf16 halves, which miss the mean by at most
    2^-9 |mean - hi| <= 2^-18 |mean|: bound (2^-16 + 2^-18) S.  Dropping the lo half errs by about 2^-10 S / sqrt(C), several
    times that.  The row means themselves (R fp32 additions and one division): (R + 1) 2^-24 sum_r |enc| / R.
  * bf16 outputs (att1, d att1 in bf16): half a bf16 ulp of ref on top.
  * Pointwise kernels propagate the allowance e of their input: sigmoid is 1/4-Lipschitz, tanh 1-Lipschitz, so the gate
    after its sigmoid gets e/4 + 2^-21, g = tanh gets e + 2^-21 (expf / tanhf are within 2 ulp, plus the add and the
    division: a few fp32 ulps of values <= 1).  c and h are checked from the kernel's own stored gates and c: only their
    roundings remain, 2^-22 (|f c_prev| + |i g|) and 2^-21 |h|.
  * Backward of the cell: dh = dhd * multiplier + (RN dcat_{t+1}) @ [W_d; W_beta; W_hh] gets the GEMM allowance plus one
    rounding.  The test carries dc in float64 beside the kernel's fp32 chain and carries its allowance E with it:
    E_dc(t) = E_dc(t+1) |f| + e_dh |o (1 - tanh^2 c)| + |dh o| (2 |tanh c| 2^-22 |tanh c| + 2^-23) + 2^-22 (|dc| + |dh o (1 -
    tanh^2 c)|), and each gate gradient gets E_dc (or e_dh for the o gate) times its Lipschitz factor plus 2^-21 of itself.
  * Cross entropy from the stored logits: the sum of V exponentials errs by at most (V + 8) 2^-24 of itself, which moves the
    log-sum-exp by that much plus 2^-23 |lse|; a probability p = exp(l - lse) then errs by p (that + 2^-24 |l - lse| + 2^-22).
  * Attention (alphas, ctx, gctx, de, d att2): |y - ref| <= 1e-5 max |ref| + 2e-8, the rule of the attention kernel tests, from
    the kernel's own att2, gate, alpha, ctx and d ctx.  d ctx and d gate_pre, which are products of the d gctx GEMM, get its
    allowance times |gate| (|ctx gate (1 - gate)|) plus a few roundings.
  * Exact: hd = hall_{t+1} x multiplier bit for bit (the injected mask, or latex_ocr_b200/philox.py's draw at the {seed, call}
    read before the call); a token fed once gets exactly its one d gates row in dptab, a token never fed exactly 0; zeros where
    the kernels write zeros (rows past a row's length in alphas, hd, row_loss, dlogits, dcat, de, d ctx; the padding columns
    [V, ldl) of logits and dlogits; d full_att.bias).

Every per-step buffer (and the bf16 mirrors, and the gradient store) is filled with a finite sentinel before the call: rows at or
past bt[t] must keep it (or hold the zeros the ragged path writes) and it must not leak into any gradient.  A finite value times a
zero d logits row is zero, so a NaN sentinel would be a false alarm.

Worst |y - ref| / bound per quantity, over every case and schedule, measured on an H100 80GB HBM3 (700 W power limit); the
whole file ran in 15 s there before the two-layer cases came (with them, this file, tests/test_gpu_lstmseq_steps.py and
tests/test_gpu_ext.py ran in 20 s together):
    bf16 roundings (a value next to a rounding midpoint nears half an ulp): att1 0.983, d att1 0.996
    pointwise and cross entropy: c 0.467, h 0.351, d gates 0.343, dc0 0.325, dlogits 0.776, dreg 0.161, gates 0.067, gate 0.068,
        row loss 0.020, loss 0.006, n_valid 0.262
    attention (1e-5 rule): alphas 0.017, ctx 0.026, gctx 0.005, de 0.057, d att2 0.106; d ctx 0.034, d gate_pre 0.033
    GEMMs and reductions (2^-16 S): out1 att2 0.014, hh 0.016, ptab 0.019, mean 0.046, h0 c0 0.039, logits 0.017, dhd 0.101,
        dh0 0.040, sreg 0.010, g_wcat1 0.038, g_bcat1 0.018, g_w_ih 0.030 / 0.027, g_b_ih 0.018, dptab 0.006, g_emb 0.041,
        g_w_fc 0.066, g_b_fc 0.023, g_w_full 0.031, g_w_enc_att 0.029, g_b_enc_att 0.004, g_w_init 0.023, g_b_init 0.012,
        d encoder_out 0.015
    layer 2 of the two-layer cases: c 0.432, h 0.279, gates 0.070, dG 0.332, dc 0.304, dh 0.037, dxt 0.037, g_w_hh 0.015,
        g_w_ih 0.021, g_b 0.013
"""
from types import SimpleNamespace

import pytest
import torch

import decoder_step_ref as ds
import lstmseq_step_ref as lr
from step_check import ACC, SENTINEL, ULPS, Checker, cell_backward_bounds, check_cell, check_gates, half_ulp_bf16, rn

pytestmark = pytest.mark.gpu

_V, _E = 500, 512
_P = 0.5

# name: (precision, impl, B, R, T, decode lengths, A = C, dropout, D)  dropout: "philox" or "mask" (injected multipliers).
# b72: steps 0 and 1 run 72 rows (the per-step GEMMs on wgmma, split-K atomics in the backward), steps 2 and 3 60 and 40 (mma.sync).
# b40: 40 rows that shrink at every step, to 33, 25 and 12 (ragged).  c1024: A = C = 1024, the widest attention and a 1024-wide K
# for the gates GEMM.  d640: the h projection has K = 640 > 512, two K slices of the mma.sync kernel with a bias.
_CASES = {
    "b8": ("bf16", "tc", 8, 44, 7, [7, 7, 6, 5, 5, 3, 2, 1], 512, "philox", 512),
    "b64": ("bf16", "tc", 64, 868, 4, [4] * 64, 512, "philox", 512),
    "b72": ("bf16", "tc", 72, 101, 4, [4] * 40 + [3] * 20 + [2] * 12, 512, "philox", 512),
    "b72mask": ("bf16", "tc", 72, 101, 4, [4] * 40 + [3] * 20 + [2] * 12, 512, "mask", 512),
    "b40": ("bf16", "tc", 40, 101, 4, [4] * 12 + [3] * 13 + [2] * 8 + [1] * 7, 512, "philox", 512),
    "c1024": ("bf16", "tc", 6, 44, 4, [4, 4, 3, 3, 2, 1], 1024, "philox", 512),
    "d640": ("bf16", "tc", 8, 44, 4, [4, 4, 4, 3, 3, 2, 2, 1], 512, "philox", 640),
    "b8fp32": ("fp32", "simt", 8, 44, 7, [7, 7, 6, 5, 5, 3, 2, 1], 512, "philox", 512),
    "b8simt": ("bf16", "simt", 8, 44, 7, [7, 7, 6, 5, 5, 3, 2, 1], 512, "philox", 512),
}

# the two-layer decoder of the extension (latex_ocr_b200/ext.py TwoLayerDecoder) on the data of a case above: phase-1 time loop,
# DecoderLayer2 over hd, phase-2 head and loss; backward phase 2, layer 2, phase 1
_TWO_LAYER = {"b8l2": "b8", "b72maskl2": "b72mask"}

# schedule -> (library options, the cases it runs)
_SCHEDULES = {
    "default": ({}, ["b8", "b64", "b72", "b72mask", "b40", "c1024", "d640", "b8fp32", "b8simt", "b8l2", "b72maskl2"]),
    "skinny_mma0": ({"skinny_mma": 0}, ["b8", "b64", "c1024"]),
    "skinny_tma0": ({"skinny_tma": 0}, ["b8", "b64"]),
    "skinny8_0": ({"skinny8": 0}, ["b72", "b8"]),
    "deterministic": ({"deterministic": 1}, ["b8", "b72", "d640", "b8l2", "b72maskl2"]),
    "deterministic_maskbits0": ({"deterministic": 1, "att_maskbits": 0}, ["b8"]),
    "wgrad256": ({"wgrad256": 1}, ["b64", "b72"]),
    "att_pipe0": ({"att_pipe": 0}, ["b8", "b72"]),
    "att_maskbits0": ({"att_maskbits": 0}, ["b8", "b64"]),
    "att_bwd_mma0": ({"att_bwd_mma": 0}, ["b8", "b64"]),
    "pdl0": ({"pdl": 0}, ["b8", "b72", "b8l2", "b72maskl2"]),
}
_PARAMS = [(s, c) for s, (_, cs) in _SCHEDULES.items() for c in cs]

_WORST = {}


def _lin(x, w, b=None):
    return ds.linear(x, w, b)


def _model(case, seed, two_layer=False):
    from latex_ocr_b200.decoder import DecoderWithAttention
    from latex_ocr_b200.ext import DecoderLayer2
    precision, impl, B, R, T, lengths, C, dropout, D = _CASES[case]
    torch.manual_seed(seed)
    dec = DecoderWithAttention(C, _E, D, _V, encoder_dim=C, dropout=_P, device="cuda", precision=precision, impl=impl)
    with torch.no_grad():
        dec.fc.bias.uniform_(-0.1, 0.1)           # init_weights zeroes it: give the bias path something to add
    layer2 = DecoderLayer2(D, device="cuda", precision=precision, impl=impl) if two_layer else None
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    enc = torch.randn(B, R, C, device="cuda", generator=g).to(dec.tdtype)
    caps = torch.randint(0, _V, (B, T + 1), device="cuda", generator=g)
    mask = None
    if dropout == "mask":
        mask = (torch.rand(B, T, D, device="cuda", generator=g) >= _P).float() / (1 - _P)
    elif dropout == "philox":
        mask = "philox"
    return dec, enc, caps, lengths, mask, layer2


def _layer2_dir(layer2, B, T):
    """Layer 2's direction as tests/test_gpu_lstmseq_steps.py's checks take it: its workspace views, weights and gradients."""
    st, n, D = layer2.store, layer2.dir.names, layer2.D
    bf = layer2.precision == "bf16"
    ent = layer2.dir.entry(T, B)
    return SimpleNamespace(v=lr.views(ent["ws"], T, B, D, D, bf), ws=ent["ws"], S=T, M=B, I=D, H=D, reverse=False, bf=bf,
                           dt=torch.bfloat16 if bf else torch.float32, w_ih=st.w(n["weight_ih"]), w_hh=st.w(n["weight_hh"]),
                           b_ih=st.f32(n["bias_ih"]), b_hh=st.f32(n["bias_hh"]), h0=None, c0=None, dh0=None, dc0=None,
                           grads={k: st.g(n[w]) for k, w in (("g_w_ih", "weight_ih"), ("g_w_hh", "weight_hh"),
                                                             ("g_b_ih", "bias_ih"), ("g_b_hh", "bias_hh"))})


_FILLED = ("out1", "hall", "call", "gates", "ctx", "gctx", "gtmp", "alphas", "hd", "row_loss", "loss", "sreg", "dlogits", "dhd",
           "dreg", "dcat", "dxh", "dc", "dctx", "de", "dptab", "datt1", "denc", "dinit", "dmean", "ptab", "mean", "att1", "bfwork")


def _run(dec, enc, caps, lengths, mask, seed, layer2=None):
    """One forward + backward from sentinel-filled buffers; returns (ws, multipliers [B][T][D] fp32, snapshots).  With
    ``layer2`` the phases run the way TwoLayerDecoder drives them, and the snapshots hold what the buffers held between them."""
    from latex_ocr_b200 import philox
    B, R, _ = enc.shape
    T = max(lengths)
    D = dec.decoder_dim
    has_do = 0 if mask is None else (2 if isinstance(mask, str) else 1)
    ws = dec.workspace(B, T, R, True)
    if has_do == 1 and ws["t"].get("dropout_mask") is None:
        ws["t"]["dropout_mask"] = torch.zeros(B, T, D, device="cuda")
    dec.store.refresh_shadow()
    dec.fill_args(ws, enc, B, T, R, has_do)          # allocates the bf16 staging on the tensor-core path
    t = ws["t"]
    for k in _FILLED:
        if k in t:
            t[k].view(torch.bfloat16 if k == "bfwork" else t[k].dtype).fill_(SENTINEL)
    t["logits"][:, :, :_V].fill_(SENTINEL)          # the padding columns keep the zeros they were allocated with
    dec.store.grad.fill_(SENTINEL)
    if layer2 is not None:
        l2 = _layer2_dir(layer2, B, T)
        for v in l2.v.values():
            v.fill_(SENTINEL)
        layer2.store.grad.fill_(SENTINEL)
    dec.seed_dropout(1000 + seed, 7)
    state = dec.dropout_state.cpu().tolist()
    snap = {}
    if layer2 is None:
        ws = dec.run_forward(enc, caps, lengths, with_loss=True, need_grad=True, dropout_mask=mask)
        dec.run_backward(ws)
    else:
        ws = dec.run_forward(enc, caps, lengths, with_loss=True, need_grad=True, dropout_mask=mask, phase=1)
        snap.update(hd1=t["hd"].clone(), logits1=t["logits"].clone(), row_loss1=t["row_loss"].clone())
        snap["l2"] = layer2.forward_inplace(t["hd"])                # hd: dropout(h1) -> h2
        dec.run_phase(ws, 2, backward=False)
        dec.run_phase(ws, 2, backward=True)                          # dhd = d h2
        snap.update(dhd2=t["dhd"].clone(), grad2=dec.store.grad.clone())
        layer2.backward_inplace(t["dhd"], snap["l2"])                # dhd: d h2 -> d dropout(h1)
        dec.run_phase(ws, 1, backward=True)
    torch.cuda.synchronize()
    if has_do == 2:
        mult = torch.from_numpy(philox.dropout_multipliers(state[0], state[1], B, T, D, _P)).cuda()
    elif has_do == 1:
        mult = mask.float()
    else:
        mult = torch.ones(B, T, D, device="cuda")
    return ws, mult, snap


def _check(ck, dec, ws, enc, caps, lengths, mult, snap=None, layer2=None):
    S = dec.store
    t_ = ws["t"]
    hd1 = snap["hd1"] if layer2 is not None else t_["hd"]               # what the time loop wrote into hd
    B, R, C = enc.shape
    T = max(lengths)
    A, D, V, E = C, dec.decoder_dim, _V, _E
    O1, G = A + C + 4 * D, 4 * D
    ldl = ws["ldl"]
    tc = dec.impl == "tc" and dec.precision == "bf16"
    act = rn if tc else (lambda x: x.double())
    fc_act = rn if (tc and ldl % 64 == 0 and D % 64 == 0) else (lambda x: x.double())
    pt_act = rn if (tc and E % 64 == 0 and G % 64 == 0 and V >= 64) else (lambda x: x.double())
    names_w = ("attention.encoder_att.weight", "attention.decoder_att.weight", "f_beta.weight", "decode_step.weight_hh",
               "embedding.weight", "decode_step.weight_ih", "init_h.weight", "init_c.weight", "fc.weight")
    p = {n: S.w(n).double() for n in names_w}
    for n in ("attention.encoder_att.bias", "attention.decoder_att.bias", "f_beta.bias", "decode_step.bias_hh", "decode_step.bias_ih",
              "init_h.bias", "init_c.bias", "fc.bias", "attention.full_att.weight"):
        p[n] = S.f32(n).double()
    wf = p["attention.full_att.weight"].reshape(-1)
    wc, bc = ds.wcat(p)
    w_ctx = p["decode_step.weight_ih"][:, E:]
    bt = [sum(1 for l in lengths if l > t) for t in range(T)]
    ragged = bt[-1] < B
    encd = enc.double()
    att1 = t_["att1"]
    att1d = att1.double()

    # ---- hoisted forward: att1, ptab, the row means, h0, c0
    ref, Sa = _lin(encd, p["attention.encoder_att.weight"], p["attention.encoder_att.bias"])
    ck.bound("att1", att1, ref, ACC * Sa + (half_ulp_bf16(ref) if att1.dtype == torch.bfloat16 else 0))
    ref, Sp = _lin(p["embedding.weight"], p["decode_step.weight_ih"][:, :E], p["decode_step.bias_ih"])
    ck.gemm("ptab", t_["ptab"], ref, Sp)
    ck.bound("mean", t_["mean"], encd.mean(1), (R + 1) * 2.0 ** -24 * encd.abs().mean(1))
    mean = t_["mean"].double()
    split = 2.0 ** -18 if (tc and C % 64 == 0 and T >= 2) else 0.0
    for k, n in ((t_["hall"][0], "init_h"), (t_["call"][0], "init_c")):
        ref, Si = _lin(mean, p[n + ".weight"], p[n + ".bias"])
        ck.bound("h0 c0", k, ref, (ACC + split) * Si)

    # ---- the forward time loop, step by step from the kernel's own inputs
    ptab = t_["ptab"].double()
    for t in range(T):
        n = bt[t]
        out1 = t_["out1"][t]
        ref, S1 = _lin(act(t_["hall"][t][:n]), wc, bc)
        ck.gemm("out1 att2", out1[:n, :A], ref[:, :A], S1[:, :A])
        ck.gemm("out1 hh", out1[:n, A + C:], ref[:, A + C:], S1[:, A + C:])
        ck.bound("out1 gate", out1[:n, A:A + C], torch.sigmoid(ref[:, A:A + C]), 0.25 * ACC * S1[:, A:A + C] + ULPS)
        att2, gate, hh = out1[:n, :A].double(), out1[:n, A:A + C].double(), out1[:n, A + C:].double()
        _, alpha, ctx, _ = ds.attention(att1d[:n], encd[:n], att2, wf, gate)
        ck.attn("alphas", t_["alphas"][:n, t], alpha)
        ck.attn("ctx", t_["ctx"][t][:n], ctx)
        ck.attn("gctx", t_["gctx"][t][:n], gate * t_["ctx"][t][:n].double())
        tok = caps[:n, t]
        pre_g, Sg = _lin(act(t_["gctx"][t][:n]), w_ctx)
        pre = pre_g + ptab[tok] + hh
        e_pre = ACC * (Sg + ptab[tok].abs() + hh.abs())
        gts = t_["gates"][t][:n]
        check_gates(ck, gts, pre, e_pre)
        i, f, g, o = gts.double().chunk(4, 1)
        check_cell(ck, t_["call"][t + 1][:n], t_["hall"][t + 1][:n], i, f, g, o, t_["call"][t][:n].double())
        ck.exact("hd", hd1[:n, t], t_["hall"][t + 1][:n] * mult[:n, t])
        # rows that stopped decoding: untouched, or the zeros of the ragged path
        for k, v in (("out1", t_["out1"][t][n:]), ("gates", t_["gates"][t][n:]), ("call", t_["call"][t + 1][n:]),
                     ("hall", t_["hall"][t + 1][n:]), ("ctx", t_["ctx"][t][n:]), ("gctx", t_["gctx"][t][n:])):
            ck.value("inactive rows of %s[%d]" % (k, t), v, SENTINEL)
        ck.value("alphas of inactive rows", t_["alphas"][n:, t], 0.0)
        ck.value("hd of inactive rows", hd1[n:, t], 0.0)

    if layer2 is not None:
        # phase 1 stops before the head; layer 2 over hd1 (its input in storage dtype) into hd, checked launch by launch
        ck.value("logits after phase 1", snap["logits1"][:, :, :V], SENTINEL)
        ck.value("row_loss after phase 1", snap["row_loss1"], SENTINEL)
        from test_gpu_lstmseq_steps import check_backward, check_forward
        ck2 = Checker(ck.tag + " layer 2")
        l2 = _layer2_dir(layer2, B, T)
        x2 = snap["l2"][0]["x"]
        ck2.exact("x", x2, hd1)
        check_forward(ck2, l2, x2, hs=t_["hd"], before_backward=False)
        check_backward(ck2, l2, snap["dhd2"], t_["dhd"])                  # d x written over d h2, after the loop read it
        ck.worst.update({"layer2 " + k: v for k, v in ck2.worst.items()})
        # phase-2 backward: the fc gradients only
        for n in S.offsets:
            if not n.startswith("fc."):
                ck.value("%s gradient after phase 2" % n, S.view(snap["grad2"], n), SENTINEL)

    # ---- head, loss (phase 2 of the two-layer decoder: over h2)
    hd = t_["hd"]
    ref, Sl = _lin(fc_act(hd), p["fc.weight"], p["fc.bias"])
    ck.gemm("logits", t_["logits"][:, :, :V], ref, Sl)
    ck.value("logits padding columns", t_["logits"][:, :, V:], 0.0)
    act_bt = torch.tensor([[t < l for t in range(T)] for l in lengths], device="cuda")           # [B][T]
    nvalid = sum(bt)
    inv_n = 1.0 / nvalid
    lg = t_["logits"][:, :, :V].double()[act_bt]
    tg = caps[:, 1:T + 1][act_bt]
    row, dl = ds.cross_entropy(lg, tg, inv_n)
    lse = torch.logsumexp(lg, -1)
    d_lse = (V + 8) * 2.0 ** -24 + 2.0 ** -23 * lse.abs()
    pr = torch.exp(lg - lse[:, None])
    d_p = pr * (d_lse[:, None] + 2.0 ** -24 * (lg - lse[:, None]).abs() + 2.0 ** -22)
    row_b = d_lse + 2.0 ** -23 * (lse.abs() + lg.gather(-1, tg[:, None])[:, 0].abs())
    rl = t_["row_loss"][:B * T].view(B, T)
    ck.bound("row_loss", rl[act_bt], row, row_b)
    ck.value("row_loss of inactive rows", rl[~act_bt], 0.0)
    ck.bound("dlogits", t_["dlogits"][:, :, :V][act_bt], dl, d_p * inv_n + 2.0 ** -23 * dl.abs())
    ck.value("dlogits of inactive rows", t_["dlogits"][~act_bt], 0.0)
    ck.value("dlogits padding columns", t_["dlogits"][:, :, V:], 0.0)
    alphas = t_["alphas"].double()
    sq, dreg = ds.regulariser(alphas, dec.alpha_c)
    Ssum = alphas.sum(1)
    e_S = (T + 1) * 2.0 ** -24 * (1 + Ssum)
    ck.bound("dreg", t_["dreg"], dreg, 2 * dec.alpha_c * e_S / (B * R) + 2.0 ** -22 * dreg.abs())
    ck.bound("loss", t_["loss"][1:2], (row.sum() * inv_n).reshape(1),
             (inv_n * row_b.sum() + ACC * inv_n * row.abs().sum()).reshape(1))
    ck.bound("loss", t_["loss"][2:3], (sq / (B * R)).reshape(1),
             ((2 * (1 - Ssum).abs() * e_S).sum() / (B * R) + ACC * sq / (B * R)).reshape(1))
    ck.bound("loss n_valid", t_["loss"][3:4], torch.full((1,), float(nvalid), dtype=torch.float64, device="cuda"),
             2.0 ** -22 * nvalid)                          # 1 / (1 / n) in fp32: two roundings
    dregk = t_["dreg"].double()
    sreg = t_["sreg"].flatten()[:B * T].view(B, T)
    ck.gemm("sreg", sreg, torch.einsum("btr,br->bt", alphas, dregk), torch.einsum("btr,br->bt", alphas.abs(), dregk.abs()))

    # ---- backward: d hd, then the time loop in reverse from the kernel's own stored values
    dlk = t_["dlogits"][:, :, :V]
    ref, Sd = fc_act(dlk) @ p["fc.weight"], fc_act(dlk).abs() @ p["fc.weight"].abs()
    ck.gemm("dhd", snap["dhd2"] if layer2 is not None else t_["dhd"], ref, Sd)
    dhd = t_["dhd"].double()                         # the two-layer decoder: layer 2's d x, read by the phase-1 backward
    multd = mult.double()
    dc = torch.zeros(B, D, dtype=torch.float64, device="cuda")
    e_dc = torch.zeros_like(dc)
    sregk = sreg.double()
    for t in range(T - 1, -1, -1):
        n = bt[t]
        dcat = t_["dcat"][t][:n]
        if t + 1 < T:
            x = act(t_["dcat"][t + 1][:n])
            dhn, e_dhn = x @ wc, ACC * (x.abs() @ wc.abs())
        else:
            dhn, e_dhn = torch.zeros(n, D, dtype=torch.float64, device="cuda"), 0.0
        dh = dhd[:n, t] * multd[:n, t] + dhn
        e_dh = e_dhn + 2.0 ** -24 * dh.abs()
        i, f, g, o = t_["gates"][t][:n].double().chunk(4, 1)
        th = torch.tanh(t_["call"][t + 1][:n].double())
        cp = t_["call"][t][:n].double()
        dG, dct, dcp = ds.cell_backward(dh, dc[:n], i, f, g, o, t_["call"][t + 1][:n].double(), cp)
        bnd, e_dct = cell_backward_bounds(e_dc[:n], e_dh, dc[:n], dh, dct, i, f, g, o, th, cp, dG)
        ck.bound("dcat gates", dcat[:, A + C:], dG, bnd)
        dc[:n], e_dc[:n] = dcp, e_dct * f.abs() + 2.0 ** -24 * dcp.abs()
        # the attention backward: d gctx = (RN dG) @ W_ih[:, E:] from the stored d gates
        x = act(dcat[:, A + C:])
        dgctx, e_dg = x @ w_ctx, ACC * (x.abs() @ w_ctx.abs())
        gate = t_["out1"][t][:n, A:A + C].double()
        ctxk = t_["ctx"][t][:n].double()
        ck.bound("dctx", t_["dctx"][t][:n], dgctx * gate, e_dg * gate + 2.0 ** -24 * (dgctx * gate).abs() + 1e-38)
        dgp = dgctx * ctxk * gate * (1 - gate)
        ck.bound("dcat gate_pre", dcat[:, A:A + C], dgp, e_dg * (ctxk * gate * (1 - gate)).abs() + ULPS * dgp.abs() + 1e-38)
        de, datt2 = ds.attention_backward_from_dctx(att1d[:n], encd[:n], t_["out1"][t][:n, :A].double(), wf, alphas[:n, t], ctxk,
                                                    t_["dctx"][t][:n].double(), dregk[:n], sregk[:n, t])
        ck.attn("de", t_["de"][:n, t], de)
        ck.attn("dcat att2", dcat[:, :A], datt2)
        if n < B:
            ck.value("dcat of inactive rows", t_["dcat"][t][n:], 0.0)
            ck.value("de of inactive rows", t_["de"][n:, t], 0.0)
            ck.value("dctx of inactive rows", t_["dctx"][t][n:], 0.0)
    x = act(t_["dcat"][0])
    ck.gemm("dinit dh0", t_["dinit"][:, :D], x @ wc, x.abs() @ wc.abs())
    ck.bound("dinit dc0", t_["dinit"][:, D:], dc, e_dc + 1e-38)

    # ---- hoisted gradients from the stored per-step values (active rows; the others are zero rows of dcat / dlogits)
    sel = act_bt.t()                                                   # [T][B]
    H = torch.stack([t_["hall"][t] for t in range(T)])[sel]
    DC = t_["dcat"][sel]
    GX = t_["gctx"][sel]
    toks = caps[:, :T].t()[sel]

    def tn(name, y, X, Y):
        ck.gemm(name, y, X.t() @ Y, X.abs().t() @ Y.abs())

    def colsum(name, y, X):
        ck.gemm(name, y, X.double().sum(0), X.double().abs().sum(0))

    gw = torch.cat([S.g("attention.decoder_att.weight"), S.g("f_beta.weight"), S.g("decode_step.weight_hh")])
    gb = torch.cat([S.g("attention.decoder_att.bias"), S.g("f_beta.bias"), S.g("decode_step.bias_hh")])
    tn("g_wcat1", gw, act(DC), act(H))
    colsum("g_bcat1", gb, DC)
    dGr = act(DC[:, A + C:])
    tn("g_w_ih ctx", S.g("decode_step.weight_ih")[:, E:], dGr, act(GX))
    colsum("g_b_ih", S.g("decode_step.bias_ih"), DC[:, A + C:])
    hit = (toks[:, None] == torch.arange(V, device="cuda")[None, :]).double()
    tn("dptab", t_["dptab"], hit, dGr)
    cnt = hit.sum(0)
    ck.value("dptab of tokens never fed", t_["dptab"][cnt == 0], 0.0)
    once = (cnt == 1).nonzero()[:, 0]
    if len(once):
        src = hit[:, once].argmax(0)
        ck.bound("dptab of tokens fed once", t_["dptab"][once], dGr[src], 0.0)
    dpt = pt_act(t_["dptab"])
    ck.gemm("g_emb", S.g("embedding.weight"), dpt @ p["decode_step.weight_ih"][:, :E], dpt.abs() @ p["decode_step.weight_ih"][:, :E].abs())
    tn("g_w_ih emb", S.g("decode_step.weight_ih")[:, :E], dpt, p["embedding.weight"])
    DL = t_["dlogits"][:, :, :V].transpose(0, 1)[sel]
    tn("g_w_fc", S.g("fc.weight"), fc_act(DL), fc_act(t_["hd"].transpose(0, 1)[sel]))
    colsum("g_b_fc", S.g("fc.bias"), DL)
    dek = t_["de"].double()
    gwf = torch.zeros(A, dtype=torch.float64, device="cuda")
    Swf = torch.zeros_like(gwf)
    da1 = torch.zeros(B, R, A, dtype=torch.float64, device="cuda")
    Sda1 = torch.zeros_like(da1)
    for t in range(T):
        pre = att1d + t_["out1"][t][:, None, :A].double()
        r = torch.relu(pre)
        gwf += torch.einsum("br,bra->a", dek[:, t], r)
        Swf += torch.einsum("br,bra->a", dek[:, t].abs(), r)
        on = (pre > 0).double()
        da1 += dek[:, t, :, None] * on
        Sda1 += dek[:, t, :, None].abs() * on
    ck.gemm("g_w_full", S.g("attention.full_att.weight").reshape(-1), gwf, Swf)
    ck.value("g_b_full", S.g("attention.full_att.bias"), 0.0)
    da1, Sda1 = da1 * wf, Sda1 * wf.abs()
    datt1 = t_["datt1"]
    ck.bound("datt1", datt1, da1, ACC * Sda1 + (half_ulp_bf16(da1) if datt1.dtype == torch.bfloat16 else 0))
    d1 = datt1.double().reshape(B * R, A)
    tn("g_w_enc_att", S.g("attention.encoder_att.weight"), d1, encd.reshape(B * R, C))
    colsum("g_b_enc_att", S.g("attention.encoder_att.bias"), d1)
    dinit = t_["dinit"].double()
    tn("g_w_init", torch.cat([S.g("init_h.weight"), S.g("init_c.weight")]), dinit, mean)
    colsum("g_b_init", torch.cat([S.g("init_h.bias"), S.g("init_c.bias")]), t_["dinit"])
    w_init = torch.cat([p["init_h.weight"], p["init_c.weight"]])
    al, dcx = act(t_["alphas"]), act(t_["dctx"].transpose(0, 1))
    We = p["attention.encoder_att.weight"]
    ref = (d1 @ We).view(B, R, C) + torch.einsum("btr,btc->brc", al, dcx) + (dinit @ w_init / R)[:, None, :]
    Sref = ((d1.abs() @ We.abs()).view(B, R, C) + torch.einsum("btr,btc->brc", al.abs(), dcx.abs())
            + (dinit.abs() @ w_init.abs() / R)[:, None, :])
    ck.gemm("d encoder_out", t_["denc"], ref, Sref)


def _outputs(dec, ws, layer2=None):
    out = [ws["t"][k].clone() for k in _FILLED if k in ws["t"]] + [ws["t"]["logits"].clone(), dec.store.grad.clone()]
    if layer2 is not None:
        B, T = ws["t"]["hd"].shape[:2]
        out += [_layer2_dir(layer2, B, T).ws.clone(), layer2.store.grad.clone()]
    return out


@pytest.mark.parametrize("schedule,case", _PARAMS, ids=["%s-%s" % sc for sc in _PARAMS])
def test_decoder_steps_vs_float64(schedule, case):
    """Every stored per-step quantity of the forward and backward time loops, the hoisted gradients and d encoder_out within
    the bounds of the module docstring of float64 from the kernel's own operands; rows that stopped decoding untouched.  Under
    "deterministic" two runs from the same state must agree bit for bit."""
    from latex_ocr_b200 import _lib
    opts, _ = _SCHEDULES[schedule]
    base = _TWO_LAYER.get(case, case)
    seed = sorted(_CASES).index(base)
    dec, enc, caps, lengths, mask, layer2 = _model(base, seed, case in _TWO_LAYER)
    with _lib.option(**opts):
        ws, mult, snap = _run(dec, enc, caps, lengths, mask, seed, layer2)
        first = _outputs(dec, ws, layer2) if "deterministic" in opts else None
        ck = Checker("%s %s" % (schedule, case))
        _check(ck, dec, ws, enc, caps, lengths, mult, snap, layer2)
        if first is not None:
            ws, _, _ = _run(dec, enc, caps, lengths, mask, seed, layer2)
            for a, b in zip(first, _outputs(dec, ws, layer2)):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "deterministic: two runs differ"
    for k, v in ck.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), v)
    print("\n%-28s %s" % (ck.tag, "  ".join("%s %.3f" % kv for kv in sorted(ck.worst.items()))))


def test_zz_worst_ratios():
    """Prints the worst |y - ref| / bound per quantity over the cases above (run after them)."""
    if not _WORST:
        pytest.skip("run with the step tests")
    print("\nworst |y - ref| / bound per quantity:")
    for k, v in sorted(_WORST.items()):
        print("  %-28s %.4f" % (k, v))
