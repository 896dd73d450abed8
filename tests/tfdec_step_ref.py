"""Float64 restatement of one step of the TensorFlow-flavour decoder (the Genthial cell, tf_decoder.Decoder, csrc/lo_tfdecoder.cuh),
split the way the kernels split it, so that a test can feed each piece the operands one kernel read and compare that kernel's
output alone.  Also the layout of the decoder's workspace (``carve``), so that a test can read every per-step quantity the kernels
store there.

Every function takes float64 tensors (any device) and returns float64 tensors.  Weights travel in a dict keyed by the TF variable
names in the TF shapes ([in][out]), as in oracle/ref_tf_model.py.  Row-vector convention: x [rows][in] @ W.

Forward of step t (E, O, D, A, C: embedding, o, LSTM, attention and image widths; K = lstm.kernel [E+O+D][4D]):
    z = [o_{t-1} | h_{t-1}] @ K[E:]                                                                   (``gates_z``)
    ptab = [embedding_table ; start_token] @ K[:E] + lstm.bias   [V+1][4D], row V = the start token    (``token_table``)
    i, j, f, o = z + ptab[token];  c = sigmoid(f + 1) c_{t-1} + sigmoid(i) tanh(j);  h = sigmoid(o) tanh(c)  (``lstm_pointwise``)
    hd = h * keep_h;  out2 = hd @ [att_h.kernel | o_W_h] = [att_h | oh]                              (``project_h``)
    e_r = tanh(att_img_r + att_h) . att_beta, alpha = softmax_r(e), ctx = sum_r alpha_r enc_r,  att_img = enc @ att_img.kernel
    o_t = tanh(ctx @ o_W_c + oh) * keep_o;  logits = o_t @ y_W_o                                      (``output``, ``logits``)
The recurrent state is (c, h, o_t): the undropped h and the dropped o.
Backward of step t (``o_backward``, ``attention_backward``, ``lstm_backward``):
    d pre_o = (d o_t from step t+1 + d logits y_W_o^T) keep_o (1 - (o_t / keep_o)^2)
    [dh_o | dctx] = d pre_o [o_W_h^T | o_W_c^T]
    s = <dctx, ctx> + sreg;  de_r = alpha_r (<dctx, enc_r> + dalpha_r - s);  d att_h = sum_r de_r beta (1 - post_r^2);
    d beta (row b) = sum_r de_r post_r,  post_r = tanh(att_img_r + att_h)
    dh = dh_rec + keep_h (dh_o + d att_h @ att_h.kernel^T)          (the recurrent path read h, the others hd)
    dc = dc_next + dh o (1 - tanh(c)^2);  dz = [dc j i (1-i), dc i (1-j^2), dc c_{t-1} f (1-f), dh tanh(c) o (1-o)];  dc_prev = dc f
    [d o_{t-1} | dh_rec(t-1)] = dz @ K[E:]^T
The hoisted gradients (``hoisted_gradients``) are sums over the steps of outer products of these per-step values.
"""
import torch


def linear(x, w, b=None):
    """(x @ w + b, |x| @ |w| + |b|): the value and the sum of the magnitudes of its terms (the scale of its rounding)."""
    y = x @ w
    s = x.abs() @ w.abs()
    if b is not None:
        y = y + b
        s = s + b.abs()
    return y, s


def w_init(p):
    """[W_c_0 | W_h_0 | W_o_0] [C][2D+O] and its bias: the initial state's one GEMM, columns in the order c | h | o."""
    return (torch.cat([p["W_c_0"], p["W_h_0"], p["W_o_0"]], 1), torch.cat([p["b_c_0"], p["b_h_0"], p["b_o_0"]], 0))


def w_cat2(p):
    """[att_h.kernel | o_W_h] [D][A+O]: the weight that projects hd onto both."""
    return torch.cat([p["att_h.kernel"], p["o_W_h"]], 1)


# ---------------------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------------------
def initial_state(p, mean):
    """(pre, s) with s = tanh(pre) [B][2D+O] = [c0 | h0 | o0] from the row means [B][C]."""
    w, b = w_init(p)
    pre = linear(mean, w, b)[0]
    return pre, torch.tanh(pre)


def token_table(p):
    """[V+1][4D]: the embedding half of the LSTM kernel for every token, row V the start token, bias included."""
    E = p["embedding_table"].shape[1]
    emb = torch.cat([p["embedding_table"], p["start_token"][None, :]], 0)
    return linear(emb, p["lstm.kernel"][:E], p["lstm.bias"])[0]


def gates_z(p, o, h):
    """z = [o | h] @ K[E:]: the recurrent half of the gate pre-activations."""
    E = p["embedding_table"].shape[1]
    return torch.cat([o, h], 1) @ p["lstm.kernel"][E:]


def lstm_pointwise(pre, c_prev):
    """(gates [B][4D] as the kernel stores them: sigmoid(i) | tanh(j) | sigmoid(f + 1) | sigmoid(o), c, h); pre = z + ptab[token]."""
    i, j, f, o = pre.chunk(4, 1)
    i, g, f, o = torch.sigmoid(i), torch.tanh(j), torch.sigmoid(f + 1.0), torch.sigmoid(o)
    c = f * c_prev + i * g
    return torch.cat([i, g, f, o], 1), c, o * torch.tanh(c)


def project_h(p, hd):
    """out2 = [att_h | oh] = hd @ [att_h.kernel | o_W_h]."""
    return hd @ w_cat2(p)


def attention(att_img, enc, att_h, beta):
    """(e, alpha, ctx): att_img [B][R][A], enc [B][R][C], att_h [B][A], beta [A]."""
    e = torch.tanh(att_img + att_h[:, None, :]) @ beta
    alpha = torch.softmax(e, dim=1)
    return e, alpha, torch.einsum("br,brc->bc", alpha, enc)


def output(p, ctx, oh, keep_o=None):
    """o_t = tanh(ctx @ o_W_c + oh) (* keep_o)."""
    o = torch.tanh(ctx @ p["o_W_c"] + oh)
    return o if keep_o is None else o * keep_o


def logits(p, o):
    return o @ p["y_W_o"]


def cross_entropy(lg, targets, inv_n):
    """(row loss, d logits) of one row block: lg [N][V], targets [N]; d logits of the mean over inv_n^-1 positions."""
    lse = torch.logsumexp(lg, dim=-1)
    row = lse - lg.gather(-1, targets[:, None])[:, 0]
    d = torch.exp(lg - lse[:, None])
    d[torch.arange(len(targets)), targets] -= 1.0
    return row, d * inv_n


# ---------------------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------------------
def o_backward(dxh_o, dologit, keep_o, o_st):
    """d pre_o of tf_o_pw_bwd_kernel: o_st is the stored (dropped) o_t; the undropped one is recovered as o_st / keep (0 where keep
    is 0, where the gradient is 0 anyway)."""
    dv = dxh_o + dologit
    o = o_st
    if keep_o is not None:
        dv = dv * keep_o
        o = torch.where(keep_o != 0, o_st / torch.where(keep_o != 0, keep_o, torch.ones_like(keep_o)), torch.zeros_like(o_st))
    return dv * (1 - o * o)


def dh_dctx(p, dpre):
    """[dh_o | dctx] = d pre_o @ [o_W_h^T | o_W_c^T]."""
    return dpre @ torch.cat([p["o_W_h"].t(), p["o_W_c"].t()], 1)


def attention_backward(att_img, enc, att_h, beta, alpha, ctx, dctx, dalpha=None, sreg=None):
    """(de [B][R], d att_h [B][A], d beta partial [B][A]) of one step; dalpha [B][R] (generic mode) with sreg [B] = <alpha, dalpha>."""
    s = (dctx * ctx).sum(-1)
    q = torch.einsum("bc,brc->br", dctx, enc)
    if dalpha is not None:
        s = s + sreg
        q = q + dalpha
    de = alpha * (q - s[:, None])
    post = torch.tanh(att_img + att_h[:, None, :])
    return de, torch.einsum("br,bra->ba", de, 1 - post * post) * beta, torch.einsum("br,bra->ba", de, post)


def dh_att(p, datt_h):
    """d att_h @ att_h.kernel^T: the attention's part of d hd."""
    return datt_h @ p["att_h.kernel"].t()


def lstm_backward(dh_rec, dh_hd, keep_h, dc_next, gates, c_prev, c):
    """(dz [B][4D], dc at this step, dc_prev) of tf_lstm_pw_bwd_kernel: dh_rec the recurrent part (it read the undropped h), dh_hd the
    attention / o-projection part (they read hd = h keep_h)."""
    D = c.shape[1]
    dh = dh_rec + (dh_hd if keep_h is None else dh_hd * keep_h)
    i, g, f, o = gates[:, :D], gates[:, D:2 * D], gates[:, 2 * D:3 * D], gates[:, 3 * D:]
    tc = torch.tanh(c)
    dc = dc_next + dh * o * (1 - tc * tc)
    dz = torch.cat([dc * g * i * (1 - i), dc * i * (1 - g * g), dc * c_prev * f * (1 - f), dh * tc * o * (1 - o)], 1)
    return dz, dc, dc * f


def dxh(p, dz):
    """[d o_{t-1} | dh_rec(t-1)] = dz @ K[E:]^T."""
    E = p["embedding_table"].shape[1]
    return dz @ p["lstm.kernel"][E:].t()


def initial_backward(d_s, s):
    """dinit = d [c0 | h0 | o0] (1 - s^2)."""
    return d_s * (1 - s * s)


def hoisted_gradients(p, enc, mean, XH, DZ, tokens, H, CTX, DOUT2, DLOGITS, O, DE, ATTH, DBETA, ALPHAS, DCTX, dinit):
    """The weight gradients and d enc the backward computes after its time loop, from the per-step values stacked over (t, b) rows
    in any common order: XH the [o_{t-1} | h_{t-1}] rows, DZ, tokens [N] the token each row consumed (V: the start token), H the hd
    rows, CTX, DOUT2 = [d att_h | d pre_o], DLOGITS, O the o_t rows; DE [B][T][R], ATTH [B][T][A], DBETA [N][A] the per-row d beta
    partials, ALPHAS [B][T][R], DCTX [B][T][C]; dinit [B][2D+O].  Keys are the TF variable names (plus dptab, datt_img, denc)."""
    V, E = p["embedding_table"].shape
    A = p["att_beta"].shape[0]
    R = enc.shape[1]
    beta = p["att_beta"]
    g = {}
    hit = (tokens[:, None] == torch.arange(V + 1, device=tokens.device)[None, :]).to(DZ.dtype)
    g["dptab"] = hit.t() @ DZ                                                      # [V+1][4D]
    ge = g["dptab"] @ p["lstm.kernel"][:E].t()
    g["embedding_table"], g["start_token"] = ge[:V], ge[V]
    emb = torch.cat([p["embedding_table"], p["start_token"][None, :]], 0)
    g["lstm.kernel"] = torch.cat([emb.t() @ g["dptab"], XH.t() @ DZ], 0)
    g["lstm.bias"] = DZ.sum(0)
    g["att_h.kernel"] = H.t() @ DOUT2[:, :A]
    g["o_W_h"] = H.t() @ DOUT2[:, A:]
    g["o_W_c"] = CTX.t() @ DOUT2[:, A:]
    g["y_W_o"] = O.t() @ DLOGITS
    g["att_beta"] = DBETA.sum(0)
    att_img = enc @ p["att_img.kernel"]
    post = torch.tanh(att_img[:, None] + ATTH[:, :, None, :])                      # [B][T][R][A]
    g["datt_img"] = beta * torch.einsum("btr,btra->bra", DE, 1 - post * post)
    g["att_img.kernel"] = torch.einsum("brc,bra->ca", enc, g["datt_img"])
    wi, _ = w_init(p)
    D = p["W_c_0"].shape[1]
    gw = mean.t() @ dinit
    gb = dinit.sum(0)
    g["W_c_0"], g["W_h_0"], g["W_o_0"] = gw[:, :D], gw[:, D:2 * D], gw[:, 2 * D:]
    g["b_c_0"], g["b_h_0"], g["b_o_0"] = gb[:D], gb[D:2 * D], gb[2 * D:]
    g["denc"] = (g["datt_img"] @ p["att_img.kernel"].t() + torch.einsum("btr,btc->brc", ALPHAS, DCTX)
                 + (dinit @ wi.t() / R)[:, None, :])
    return g


# ---------------------------------------------------------------------------------------------------------------------------------
# the pieces chained over T steps: what tests/test_tfdec_step_ref.py checks against oracle/ref_tf_model.py
# ---------------------------------------------------------------------------------------------------------------------------------
def tokens_consumed(formula, V, fed=None):
    """[B][T]: the token step t consumes: V (the start token) at t = 0, else formula[b][t-1], or fed[b][t-1] when sampling."""
    src = formula if fed is None else fed
    return torch.cat([torch.full_like(src[:, :1], V), src[:, :-1]], 1)


def chained(p, enc, formula, lengths, keep_h=None, keep_o=None, fed=None):
    """Forward, masked cross entropy and backward of a whole sequence from the pieces above: (loss, per-step values, gradients).
    formula [B][T] are the targets; the tokens consumed are formula's (or fed's, sampling) shifted by one behind the start token."""
    B, R, C = enc.shape
    T = formula.shape[1]
    V, E = p["embedding_table"].shape
    D = p["W_c_0"].shape[1]
    A = p["att_beta"].shape[0]
    beta = p["att_beta"]
    kh = (lambda t: None) if keep_h is None else (lambda t: keep_h[:, t])
    ko = (lambda t: None) if keep_o is None else (lambda t: keep_o[:, t])
    att_img = enc @ p["att_img.kernel"]
    mean = enc.mean(1)
    _, s0 = initial_state(p, mean)
    c, h, o = s0[:, :D], s0[:, D:2 * D], s0[:, 2 * D:]
    ptab = token_table(p)
    tok = tokens_consumed(formula, V, fed)
    s = {k: [] for k in ("xh", "c_prev", "gates", "c", "h", "hd", "out2", "alpha", "ctx", "o")}
    for t in range(T):
        xh = torch.cat([o, h], 1)
        gt, c2, h2 = lstm_pointwise(gates_z(p, o, h) + ptab[tok[:, t]], c)
        hd = h2 if keep_h is None else h2 * kh(t)
        out2 = project_h(p, hd)
        _, alpha, ctx = attention(att_img, enc, out2[:, :A], beta)
        o2 = output(p, ctx, out2[:, A:], ko(t))
        for k, v in zip(s, (xh, c, gt, c2, h2, hd, out2, alpha, ctx, o2)):
            s[k].append(v)
        c, h, o = c2, h2, o2
    O_ = torch.stack(s["o"], 0)                                                    # [T][B][O]
    lg = logits(p, O_)                                                             # time-major [T][B][V]
    valid = (torch.arange(T, device=enc.device)[:, None] < lengths.to(enc.device)[None, :])        # [T][B]
    inv_n = 1.0 / float(valid.sum())
    row, dl = cross_entropy(lg.reshape(T * B, V), formula.t().reshape(-1), inv_n)
    vf = valid.reshape(-1).to(lg.dtype)
    loss = (row * vf).sum() * inv_n
    dlogits = (dl * vf[:, None]).view(T, B, V)
    dologit = dlogits @ p["y_W_o"].t()
    dxh_o = torch.zeros_like(o)
    dh_rec = torch.zeros_like(h)
    dc = torch.zeros_like(c)
    st = {k: [None] * T for k in ("dpre", "dctx", "de", "datt_h", "dbeta", "dz")}
    for t in range(T - 1, -1, -1):
        dpre = o_backward(dxh_o, dologit[t], ko(t), s["o"][t])
        dhc = dh_dctx(p, dpre)
        dctx = dhc[:, D:]
        de, datt_h, dbeta = attention_backward(att_img, enc, s["out2"][t][:, :A], beta, s["alpha"][t], s["ctx"][t], dctx)
        dz, _, dc = lstm_backward(dh_rec, dhc[:, :D] + dh_att(p, datt_h), kh(t), dc, s["gates"][t], s["c_prev"][t], s["c"][t])
        dx = dxh(p, dz)
        dxh_o, dh_rec = dx[:, :o.shape[1]], dx[:, o.shape[1]:]
        for k, v in zip(st, (dpre, dctx, de, datt_h, dbeta, dz)):
            st[k][t] = v
    dinit = initial_backward(torch.cat([dc, dh_rec, dxh_o], 1), s0)

    def rows(v):
        return torch.cat(v, 0)                                                     # time-major (t, b) rows
    g = hoisted_gradients(p, enc, mean, rows(s["xh"]), rows(st["dz"]), tok.t().reshape(-1), rows(s["hd"]), rows(s["ctx"]),
                          torch.cat([rows(st["datt_h"]), rows(st["dpre"])], 1), dlogits.reshape(T * B, V), rows(s["o"]),
                          torch.stack(st["de"], 1), torch.stack([x[:, :A] for x in s["out2"]], 1), rows(st["dbeta"]),
                          torch.stack(s["alpha"], 1), torch.stack(st["dctx"], 1), dinit)
    return loss, dict(s, logits=lg, dlogits=dlogits, dinit=dinit, s0=s0, **st), g


# ---------------------------------------------------------------------------------------------------------------------------------
# the workspace: tf_carve (csrc/lo_tfdecoder.cuh) restated
# ---------------------------------------------------------------------------------------------------------------------------------
def attention_workspace_bytes(B, C):
    """lo_attention_workspace_bytes for B <= 1024 (tests/test_attention_workspace_layout.py): 4096 + the split partials."""
    return 4096 + B * 16 * (C + 2) * 4


def carve(B, T, R, C, A, D, O, E, V, ldl, bf16):
    """(views, end): name -> (byte offset, dtype, shape) of every region of the workspace up to ``sreg``, and the offset where the
    next region (the ragged decode's CTA map, which depends on B only) starts.  Training layout: rows_per_img = 1."""
    es = 2 if bf16 else 4
    XH, G, N2 = O + D, 4 * D, A + O
    Vl = ldl or V
    TB, T1B = T * B, (T + 1) * B
    f32, b16, wdt = torch.float32, torch.bfloat16, (torch.bfloat16 if bf16 else torch.float32)
    plan = [("att_img", wdt, (B, R, A)), ("datt_img", wdt, (B, R, A)), ("dbeta_acc", f32, (B, A)),
            ("ptab", f32, (V + 1, G)), ("dptab", f32, (V + 1, G)), ("xh", f32, (T + 1, B, XH)), ("call", f32, (T + 1, B, D)),
            ("gates", f32, (T, B, G)), ("ztmp", f32, (B, G)), ("out2", f32, (T, B, N2)), ("ctx", f32, (T, B, C)), ("oc", f32, (B, O)),
            ("dologit", f32, (T, B, O)), ("dout2", f32, (T, B, N2)), ("dhc", f32, (B, D + C)), ("dz", f32, (T, B, G)),
            ("dxh", f32, (B, XH)), ("dc", f32, (B, D)), ("de", f32, (B, T, R)), ("dctx", f32, (T, B, C)), ("mean", f32, (B, C)),
            ("initpre", f32, (B, 2 * D + O)), ("sinit", f32, (B, 2 * D + O)), ("dinit", f32, (B, 2 * D + O)),
            ("dmean", f32, (B, C)), ("dlogits", f32, (T, B, Vl)), ("row_loss", f32, (T, B)), ("gtmp", f32, (B, max(XH, D)))]
    if bf16:
        plan += [("xh_bf", b16, (T + 1, B, XH)), ("ctx_bf", b16, (T, B, C)), ("dout2_bf", b16, (T, B, N2)), ("dz_bf", b16, (T, B, G)),
                 ("dlogits_bf", b16, (T, B, Vl))]
    plan += [("hd", f32, (T, B, D))]
    if bf16:
        plan += [("hd_bf", b16, (T, B, D))]
    plan += [("wb4", wdt, (D + C, O)), ("wb5", wdt, (D, A)), ("wb6", wdt, (XH, G)), ("wbY", wdt, (O, Vl)), ("wimgT", wdt, (C, A)),
             ("attwork", torch.uint8, (attention_workspace_bytes(B, C),)), ("next_tok", torch.int64, (B,)),
             ("finished", torch.int32, (B,)), ("parent_rows", torch.int32, (B,)), ("sreg", f32, (B, T))]
    views, off = {}, 0
    for name, dt, shape in plan:
        views[name] = (off, dt, shape)
        n = dt.itemsize
        for x in shape:
            n *= x
        off += (n + 255) // 256 * 256
    return views, off


def views_of(ws, layout):
    """name -> tensor view of the uint8 workspace ``ws`` for the layout of ``carve``."""
    out = {}
    for name, (off, dt, shape) in layout.items():
        n = dt.itemsize
        for x in shape:
            n *= x
        out[name] = ws[off:off + n].view(dt).view(shape)
    return out
