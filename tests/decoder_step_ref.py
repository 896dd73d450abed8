"""Float64 restatement of one step of the torch-flavour decoder (DecoderWithAttention, csrc/lo_decoder.cu), split the way the
kernels split it, so that a test can feed each piece the operands one kernel read and compare that kernel's output alone.

Every function takes float64 tensors (any device) and returns float64 tensors.  Weights travel in a dict keyed by the
reference's ``state_dict`` names, as in oracle/ref_model.py.  Row-vector convention: x [rows][in] @ W^T.

Forward of step t (rows still decoding):
    out1 = h_{t-1} @ [W_d; W_beta; W_hh]^T + [b_d; b_beta; b_hh] = [att2 | gate_pre | hh]        (one GEMM, ``project``)
    alpha = softmax_r(relu(att1_r + att2) . w_full), ctx = sum_r alpha_r enc_r, gate = sigmoid(gate_pre), gctx = gate * ctx
    pre = gctx @ W_ih[:, E:]^T + ptab[token] + hh,  ptab = emb @ W_ih[:, :E]^T + b_ih               (``cell``)
    i, f, o = sigmoid, g = tanh;  c = f c_{t-1} + i g;  h = o tanh(c);  hd = h * dropout multiplier
    logits = hd @ W_fc^T + b_fc
Backward of step t (``cell_backward``, ``attention_backward``):
    dh = dhd * multiplier + dh_next;  dc = dc_next + dh o (1 - tanh(c)^2)
    dG = [dc g i (1-i), dc c_{t-1} f (1-f), dc i (1-g^2), dh tanh(c) o (1-o)];  dc_prev = dc f
    dgctx = dG @ W_ih[:, E:];  dctx = dgctx gate;  dgp = dgctx ctx gate (1-gate)
    s = <dctx, ctx> + sreg;  de_r = alpha_r (<dctx, enc_r> + dreg_r - s);  datt2 = w_full * sum_r de_r [att1_r + att2 > 0]
    dcat = [datt2 | dgp | dG];  dh_prev = dcat @ [W_d; W_beta; W_hh]
The hoisted gradients (``hoisted_gradients``) are sums over the steps of outer products of these per-step values.
"""
import torch


def wcat(p):
    """The packed [W_d; W_beta; W_hh] block ([A + C + 4D][D]) and its bias: the weight of the per-step projection."""
    return (torch.cat([p["attention.decoder_att.weight"], p["f_beta.weight"], p["decode_step.weight_hh"]], 0),
            torch.cat([p["attention.decoder_att.bias"], p["f_beta.bias"], p["decode_step.bias_hh"]], 0))


def linear(x, w, b=None):
    """(x @ w^T + b, |x| @ |w|^T + |b|): the value and the sum of the magnitudes of its terms (the scale of its rounding)."""
    y = x @ w.t()
    s = x.abs() @ w.abs().t()
    if b is not None:
        y = y + b
        s = s + b.abs()
    return y, s


# ---------------------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------------------
def init_state(p, mean):
    """h0, c0 of init_hidden_state from the row means [B][C]."""
    return linear(mean, p["init_h.weight"], p["init_h.bias"])[0], linear(mean, p["init_c.weight"], p["init_c.bias"])[0]


def proj_table(p, C):
    """The embedding -> gate table [V][4D] = emb @ W_ih[:, :E]^T + b_ih (bias_hh travels with the projection of h)."""
    E = p["decode_step.weight_ih"].shape[1] - C
    return linear(p["embedding.weight"], p["decode_step.weight_ih"][:, :E], p["decode_step.bias_ih"])[0]


def project(p, h):
    """out1 before the attention's in-place sigmoid: [att2 | gate_pre | hh] = h @ wcat^T + bcat."""
    w, b = wcat(p)
    return linear(h, w, b)[0]


def attention(att1, enc, att2, wf, gate):
    """(e, alpha, ctx, gctx) of one step: att1 [B][R][A], enc [B][R][C], att2 [B][A], wf [A], gate [B][C] (after the sigmoid).
    The score has no full_att bias: softmax does not see it."""
    e = torch.relu(att1 + att2[:, None, :]) @ wf
    alpha = torch.softmax(e, dim=1)
    ctx = torch.einsum("br,brc->bc", alpha, enc)
    return e, alpha, ctx, gate * ctx


def cell(p, gctx, table_rows, hh, c_prev):
    """(pre, i, f, g, o, c, h) of the LSTM cell; table_rows = ptab[token] [B][4D], hh the recurrent block of out1."""
    C = gctx.shape[1]
    E = p["decode_step.weight_ih"].shape[1] - C
    pre = linear(gctx, p["decode_step.weight_ih"][:, E:])[0] + table_rows + hh
    i, f, g, o = pre.chunk(4, dim=1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c = f * c_prev + i * g
    return pre, i, f, g, o, c, o * torch.tanh(c)


def head(p, hd):
    return linear(hd, p["fc.weight"], p["fc.bias"])[0]


def cross_entropy(logits, targets, inv_n):
    """(row loss, d logits) of one row block: logits [N][V], targets [N]; d logits of the mean over inv_n^-1 positions."""
    lse = torch.logsumexp(logits, dim=-1)
    row = lse - logits.gather(-1, targets[:, None])[:, 0]
    d = torch.exp(logits - lse[:, None])
    d[torch.arange(len(targets)), targets] -= 1.0
    return row, d * inv_n


def regulariser(alphas, alpha_c):
    """(sum over b, r of (1 - sum_t alpha)^2, d alpha [B][R] of alpha_c times its mean): alphas [B][T][R]."""
    B, _, R = alphas.shape
    d = 1.0 - alphas.sum(dim=1)
    return (d * d).sum(), -2.0 * alpha_c * d / (B * R)


# ---------------------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------------------
def cell_backward(dh, dc_next, i, f, g, o, c, c_prev):
    """(dG [B][4D], dc at this step, dc_prev) of the cell given dh (incl. the head's part) and the carried dc."""
    tc = torch.tanh(c)
    dc = dc_next + dh * o * (1 - tc * tc)
    dG = torch.cat([dc * g * i * (1 - i), dc * c_prev * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], dim=1)
    return dG, dc, dc * f


def context_grad(p, dG):
    """d gctx = dG @ W_ih[:, E:]."""
    C = p["f_beta.weight"].shape[0]
    E = p["decode_step.weight_ih"].shape[1] - C
    return dG @ p["decode_step.weight_ih"][:, E:]


def attention_backward(att1, enc, att2, gate, wf, alpha, ctx, dgctx, dreg, sreg):
    """(dctx, dgp, de, datt2) of one step; dreg [B][R] the regulariser's d alpha, sreg [B] = <alpha, dreg>."""
    dctx = dgctx * gate
    dgp = dgctx * ctx * gate * (1 - gate)
    return (dctx, dgp) + attention_backward_from_dctx(att1, enc, att2, wf, alpha, ctx, dctx, dreg, sreg)


def attention_backward_from_dctx(att1, enc, att2, wf, alpha, ctx, dctx, dreg, sreg):
    """(de, datt2) from d ctx."""
    s = (dctx * ctx).sum(-1) + sreg
    de = alpha * (torch.einsum("bc,brc->br", dctx, enc) + dreg - s[:, None])
    datt2 = wf * torch.einsum("br,bra->ba", de, ((att1 + att2[:, None, :]) > 0).to(de.dtype))
    return de, datt2


def hidden_grad(p, dcat):
    """dh_prev = [datt2 | dgp | dG] @ [W_d; W_beta; W_hh]."""
    return dcat @ wcat(p)[0]


def hoisted_gradients(p, enc, att1, mean, H, GCTX, HD, DLOGITS, DCAT, DE, ATT2, ALPHAS, DCTX, tokens, dinit):
    """The weight gradients and d enc the backward computes after its time loop, from the per-step values stacked over
    (b, t) rows in any common order: H the h_prev rows, GCTX, HD, DLOGITS [N][V], DCAT [N][A+C+4D], tokens [N] (-1: a row that
    feeds nothing).  DE [B][T][R], ATT2 [B][T][A], ALPHAS [B][T][R], DCTX [B][T][C]; dinit = [dh0 | dc0]."""
    C = enc.shape[2]
    A = att1.shape[2]
    V, E = p["embedding.weight"].shape
    D = H.shape[1]
    R = enc.shape[1]
    wf = p["attention.full_att.weight"].reshape(-1)
    g = {}
    g["wcat1"] = DCAT.t() @ H
    g["bcat1"] = DCAT.sum(0)
    dG = DCAT[:, A + C:]
    g["w_ih_ctx"] = dG.t() @ GCTX
    g["b_ih"] = dG.sum(0)
    hit = (tokens[:, None] == torch.arange(V, device=tokens.device)[None, :]).to(dG.dtype)
    g["dptab"] = hit.t() @ dG
    g["emb"] = g["dptab"] @ p["decode_step.weight_ih"][:, :E]
    g["w_ih_emb"] = g["dptab"].t() @ p["embedding.weight"]
    g["w_fc"] = DLOGITS.t() @ HD
    g["b_fc"] = DLOGITS.sum(0)
    pre = att1[:, None] + ATT2[:, :, None, :]                                      # [B][T][R][A]
    g["datt1"] = wf * torch.einsum("btr,btra->bra", DE, (pre > 0).to(DE.dtype))
    g["w_full"] = torch.einsum("btr,btra->a", DE, torch.relu(pre))
    g["w_enc_att"] = torch.einsum("bra,brc->ac", g["datt1"], enc)
    g["b_enc_att"] = g["datt1"].sum((0, 1))
    g["w_init"] = dinit.t() @ mean                                                 # [2D][C]: init_h rows, then init_c
    g["b_init"] = dinit.sum(0)
    w_init = torch.cat([p["init_h.weight"], p["init_c.weight"]], 0)
    g["denc"] = (g["datt1"] @ p["attention.encoder_att.weight"] + torch.einsum("btr,btc->brc", ALPHAS, DCTX)
                 + (dinit @ w_init / R)[:, None, :])
    return g


# ---------------------------------------------------------------------------------------------------------------------------------
# the pieces chained over T steps (every row decodes T steps): what tests/test_decoder_step_ref.py checks against oracle/ref_model.py
# ---------------------------------------------------------------------------------------------------------------------------------
def chained(p, enc, caps, T, mult=None, alpha_c=1.0):
    """Forward and backward of a whole sequence from the pieces above: (loss, per-step values, hoisted gradients)."""
    B, R, C = enc.shape
    A = p["attention.encoder_att.weight"].shape[0]
    V = p["fc.weight"].shape[0]
    wf = p["attention.full_att.weight"].reshape(-1)
    att1 = linear(enc, p["attention.encoder_att.weight"], p["attention.encoder_att.bias"])[0]
    mean = enc.mean(1)
    h, c = init_state(p, mean)
    ptab = proj_table(p, C)
    s = {k: [] for k in ("h_prev", "c_prev", "att2", "gate", "alpha", "ctx", "gctx", "i", "f", "g", "o", "c", "h", "hd")}
    for t in range(T):
        out1 = project(p, h)
        att2, gate = out1[:, :A], torch.sigmoid(out1[:, A:A + C])
        _, alpha, ctx, gctx = attention(att1, enc, att2, wf, gate)
        _, i, f, g, o, c2, h2 = cell(p, gctx, ptab[caps[:, t]], out1[:, A + C:], c)
        hd = h2 if mult is None else h2 * mult[:, t]
        for k, v in zip(s, (h, c, att2, gate, alpha, ctx, gctx, i, f, g, o, c2, h2, hd)):
            s[k].append(v)
        h, c = h2, c2
    HD = torch.stack(s["hd"], 1)                                                   # [B][T][D]
    logits = head(p, HD)
    alphas = torch.stack(s["alpha"], 1)
    inv_n = 1.0 / (B * T)
    row, dlogits = cross_entropy(logits.reshape(B * T, V), caps[:, 1:T + 1].reshape(-1), inv_n)
    sq, dreg = regulariser(alphas, alpha_c)
    loss = row.sum() * inv_n + alpha_c * sq / (B * R)
    dlogits = dlogits.view(B, T, V)
    dhd = dlogits @ p["fc.weight"]
    sreg = torch.einsum("btr,br->bt", alphas, dreg)
    dh_next = torch.zeros_like(h)
    dc_next = torch.zeros_like(c)
    dcat, de, dctx = [None] * T, [None] * T, [None] * T
    for t in range(T - 1, -1, -1):
        dh = dhd[:, t] * (1.0 if mult is None else mult[:, t]) + dh_next
        dG, _, dc_next = cell_backward(dh, dc_next, s["i"][t], s["f"][t], s["g"][t], s["o"][t], s["c"][t], s["c_prev"][t])
        dctx[t], dgp, de[t], datt2 = attention_backward(att1, enc, s["att2"][t], s["gate"][t], wf, s["alpha"][t], s["ctx"][t],
                                                        context_grad(p, dG), dreg, sreg[:, t])
        dcat[t] = torch.cat([datt2, dgp, dG], 1)
        dh_next = hidden_grad(p, dcat[t])
    dinit = torch.cat([dh_next, dc_next], 1)

    def rows(k):
        return torch.stack(s[k], 1).reshape(B * T, -1)
    g = hoisted_gradients(p, enc, att1, mean, rows("h_prev"), rows("gctx"), HD.reshape(B * T, -1), dlogits.reshape(B * T, V),
                          torch.stack(dcat, 1).reshape(B * T, -1), torch.stack(de, 1), torch.stack(s["att2"], 1), alphas,
                          torch.stack(dctx, 1), caps[:, :T].reshape(-1), dinit)
    return loss, dict(s, logits=logits, alphas=alphas, dcat=dcat, de=de, dctx=dctx, dinit=dinit), g


def as_reference_grads(p, g):
    """The hoisted gradients in the reference's ``state_dict`` layout (oracle/ref_model.py:decoder_backward_manual's dict)."""
    A = p["attention.encoder_att.weight"].shape[0]
    C = p["f_beta.weight"].shape[0]
    D = p["init_h.weight"].shape[0]
    out = {
        "attention.decoder_att.weight": g["wcat1"][:A], "attention.decoder_att.bias": g["bcat1"][:A],
        "f_beta.weight": g["wcat1"][A:A + C], "f_beta.bias": g["bcat1"][A:A + C],
        "decode_step.weight_hh": g["wcat1"][A + C:], "decode_step.bias_hh": g["bcat1"][A + C:],
        "decode_step.weight_ih": torch.cat([g["w_ih_emb"], g["w_ih_ctx"]], 1), "decode_step.bias_ih": g["b_ih"],
        "embedding.weight": g["emb"], "fc.weight": g["w_fc"], "fc.bias": g["b_fc"],
        "attention.full_att.weight": g["w_full"].reshape(1, -1),
        "attention.encoder_att.weight": g["w_enc_att"], "attention.encoder_att.bias": g["b_enc_att"],
        "init_h.weight": g["w_init"][:D], "init_c.weight": g["w_init"][D:], "init_h.bias": g["b_init"][:D],
        "init_c.bias": g["b_init"][D:],
    }
    return out
