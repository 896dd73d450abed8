"""Float64 restatement of the sequence LSTM (lo_lstm_seq_forward / lo_lstm_seq_backward, csrc/lo_lstmseq.cuh), split the way the
kernels split it, so that a test can feed each piece the operands one launch read and compare that launch's output alone.

Every function takes float64 tensors (any device) and returns float64 tensors.  Row-vector convention: x [rows][in] @ W^T, gate
order i, f, g, o (nn.LSTM).  Internally everything is ordered by processing step p: t(p) = p, or S-1-p when ``reverse``.

Forward (``gather``, ``input_projection``, ``recurrent``, ``cell_forward``):
    xt[p] = x[:, t(p)];  pre[p] = xt[p] W_ih^T + (b_ih + b_hh)          (one hoisted GEMM over every step)
    pre[p] += h[p] W_hh^T                                                (slot p of h holds h_{p-1}; slot 0 h0 or zeros)
    i, f, o = sigmoid, g = tanh;  c[p+1] = f c[p] + i g;  h[p+1] = o tanh(c[p+1])
Backward of step p (``cell_backward``, ``carried``), as seq_lstm_pw_bwd_kernel orders it:
    dh = dhs[t(p)] + carried;  dct = dc + dh o (1 - tanh(c)^2)
    dG = [dct g i (1-i), dct c[p] f (1-f), dct i (1-g^2), dh tanh(c) o (1-o)];  dc <- dct f;  carried <- dG W_hh
Hoisted (``hoisted_gradients``, ``scatter``): g_w_hh = dG^T h[0..S-1], g_w_ih = dG^T xt, g_b_ih = g_b_hh = sum of dG rows,
dxt = dG W_ih, scattered to dx[:, t(p)] (or added onto it).
"""
import torch


def order(S, reverse):
    """t(p) for p = 0..S-1."""
    return [S - 1 - p if reverse else p for p in range(S)]


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
def gather(x, reverse):
    """x [M][S][I] (the caller's (m, t) elements) -> xt [S][M][I] in processing order."""
    return x.transpose(0, 1)[order(x.shape[1], reverse)]


def input_projection(xt, w_ih, b_ih, b_hh):
    """(pre, magnitude sum) of the hoisted product: xt [..][I] -> [..][4H], with the summed bias."""
    return linear(xt, w_ih, b_ih + b_hh)


def recurrent(h_prev, w_hh):
    """(h_prev W_hh^T, magnitude sum): the per-step product added onto the hoisted pre-activations."""
    return linear(h_prev, w_hh)


def cell_forward(pre, c_prev):
    """(i, f, g, o, c, h) of the cell from the pre-activations [..][4H] and c_prev."""
    i, f, g, o = pre.chunk(4, dim=-1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c = f * c_prev + i * g
    return i, f, g, o, c, o * torch.tanh(c)


# ---------------------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------------------
def cell_backward(dhs, carried, dc, i, f, g, o, c, c_prev):
    """(dh, dct, dG [..][4H], dc_prev) of one step: dhs the caller's d h at t(p) (0 without), carried = dG_{p+1} W_hh, dc the
    carried d c."""
    dh = dhs + carried
    tc = torch.tanh(c)
    dct = dc + dh * o * (1 - tc * tc)
    dG = torch.cat([dct * g * i * (1 - i), dct * c_prev * f * (1 - f), dct * i * (1 - g * g), dh * tc * o * (1 - o)], dim=-1)
    return dh, dct, dG, dct * f


def carried(dG, w_hh):
    """d h_{p-1} = dG_p W_hh."""
    return dG @ w_hh


def hoisted_gradients(DG, HPREV, XT, w_ih):
    """The gradients computed after the time loop from the per-step values stacked over (p, m) rows: DG [N][4H], HPREV [N][H]
    (h slots 0..S-1), XT [N][I].  g_b is the bias gradient of both b_ih and b_hh; dxt [N][I]."""
    return {"g_w_hh": DG.t() @ HPREV, "g_w_ih": DG.t() @ XT, "g_b": DG.sum(0), "dxt": DG @ w_ih}


def scatter(dxt, reverse, base=None):
    """dxt [S][M][I] in processing order -> dx [M][S][I] (added onto ``base`` when given: dx_accumulate)."""
    S = dxt.shape[0]
    dx = torch.empty_like(dxt.transpose(0, 1))
    dx[:, order(S, reverse)] = dxt.transpose(0, 1)
    return dx if base is None else base + dx


# ---------------------------------------------------------------------------------------------------------------------------------
# the pieces chained over S steps: what tests/test_lstmseq_step_ref.py checks against oracle/ref_ext.py and torch.nn.LSTM
# ---------------------------------------------------------------------------------------------------------------------------------
def chained(x, w_ih, w_hh, b_ih, b_hh, reverse=False, h0=None, c0=None, dhs=None, dx_base=None):
    """Forward and backward of one direction: x [M][S][I], dhs [M][S][H] (None: zeros).  Returns (hs [M][S][H], per-step values
    in processing order, gradients {g_w_ih, g_w_hh, g_b, dx, dh0, dc0})."""
    M, S, _ = x.shape
    H = w_hh.shape[1]
    ts = order(S, reverse)
    xt = gather(x, reverse)
    pre = input_projection(xt, w_ih, b_ih, b_hh)[0]
    h = [h0 if h0 is not None else x.new_zeros(M, H)]
    c = [c0 if c0 is not None else x.new_zeros(M, H)]
    gates = []
    for p in range(S):
        i, f, g, o, cn, hn = cell_forward(pre[p] + recurrent(h[p], w_hh)[0], c[p])
        gates.append((i, f, g, o))
        h.append(hn)
        c.append(cn)
    hs = torch.stack(h[1:], 1)[:, ts]              # processing order p -> time t(p) (the map is its own inverse)
    dG = [None] * S
    cr = x.new_zeros(M, H)
    dc = x.new_zeros(M, H)
    for p in range(S - 1, -1, -1):
        d = dhs[:, ts[p]] if dhs is not None else 0.0
        _, _, dG[p], dc = cell_backward(d, cr, dc, *gates[p], c[p + 1], c[p])
        cr = carried(dG[p], w_hh)
    DG = torch.stack(dG)
    g = hoisted_gradients(DG.reshape(S * M, -1), torch.stack(h[:S]).reshape(S * M, H), xt.reshape(S * M, -1), w_ih)
    g["dx"] = scatter(g.pop("dxt").view(S, M, -1), reverse, dx_base)
    g["dh0"], g["dc0"] = cr, dc
    return hs, {"xt": xt, "gates": gates, "h": h, "c": c, "dG": dG}, g


# ---------------------------------------------------------------------------------------------------------------------------------
# the workspace carve (seq_carve) as named views
# ---------------------------------------------------------------------------------------------------------------------------------
def carve(S, M, I, H, bf16):
    """({name: (byte offset, dtype, shape)}, end offset) of the workspace regions in the library's order, each padded to 256
    bytes.  The bf16 mirrors exist in bf16 storage only; xt, whhT and wihT are in the storage dtype."""
    st = torch.bfloat16 if bf16 else torch.float32
    G = 4 * H
    regions = [("xt", st, (S, M, I)), ("gates", torch.float32, (S, M, G)), ("h", torch.float32, (S + 1, M, H)),
               ("c", torch.float32, (S + 1, M, H))]
    if bf16:
        regions.append(("h_bf", torch.bfloat16, (S + 1, M, H)))
    regions.append(("dG", torch.float32, (S, M, G)))
    if bf16:
        regions.append(("dG_bf", torch.bfloat16, (S, M, G)))
    regions += [("dh", torch.float32, (M, H)), ("dc", torch.float32, (M, H)), ("dxt", torch.float32, (S, M, I)),
                ("whhT", st, (H, G)), ("wihT", st, (I, G)), ("bsum", torch.float32, (G,))]
    views, off = {}, 0
    for name, dt, shape in regions:
        n = 1
        for s in shape:
            n *= s
        views[name] = (off, dt, shape)
        off += (n * (2 if dt == torch.bfloat16 else 4) + 255) // 256 * 256
    return views, off


def views(ws, S, M, I, H, bf16):
    """{name: tensor view} of a uint8 workspace tensor."""
    v, _ = carve(S, M, I, H, bf16)
    out = {}
    for name, (off, dt, shape) in v.items():
        n = 1
        for s in shape:
            n *= s
        es = 2 if dt == torch.bfloat16 else 4
        out[name] = ws[off:off + n * es].view(dt).view(shape)
    return out
