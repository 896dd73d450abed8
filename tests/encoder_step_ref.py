"""Float64 restatement of the encoder's launches (EncoderCNN.forward_raw / backward_raw, csrc/lo_conv.cu), one function per
launch, on the kernels' layouts: feature maps NHWC, 3 x 3 weights [Cout][3][3][Cin], the strided conv's weights [Cout][R*S*C]
(tap-major, as im2col lays out its columns).

Every function that sums returns, beside each sum, S: the float64 sum of the magnitudes of its terms, so a caller can bound
an fp32 evaluation of the same sum element by element.  Inputs may live on any device and have any dtype; everything is
computed in float64.  tests/test_encoder_step_ref.py chains these pieces and checks them against oracle/ref_model.py;
tests/test_gpu_encoder_steps.py compares each kernel with its piece on the operands the kernel read."""
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_weight


def _nchw(x):
    return x.double().permute(0, 3, 1, 2).contiguous()


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------------------------------
# conv1 (Cin = 1) + bias + ReLU + 2 x 2 max-pool, and its weight gradient routed by the arg-max / ReLU codes
# ------------------------------------------------------------------------------------------------------------------------
def pixels(img, scale=1.0, offset=0.0):
    """The pixels conv1 reads, [N][H][W] float64: fl32(img * scale + offset), the kernel's one fmaf per pixel (exact for
    scale 1 / offset 0 and for integer pixels under the TF normalisation 1/128, -1)."""
    x = img.double().reshape(img.shape[0], img.shape[-2], img.shape[-1])
    return (x * scale + offset).float().double()


def conv1_windows(x, w, b):
    """conv1 + bias at the four conv positions of every 2 x 2 pool window.  x [N][H][W] pixels, w [64][1][3][3] (or [64][9]),
    b [64].  Returns (v, S), both [N][H/2][W/2][64][4] with the window position py * 2 + px last (the kernels' scan order)."""
    N, H, W = x.shape
    Hp, Wp = H // 2, W // 2
    w4 = w.double().reshape(64, 1, 3, 3)
    bd = b.double()
    v = F.conv2d(x[:, None], w4, bd, padding=1)[:, :, :2 * Hp, :2 * Wp]
    S = F.conv2d(x.abs()[:, None], w4.abs(), bd.abs(), padding=1)[:, :, :2 * Hp, :2 * Wp]

    def win(t):
        return t.reshape(N, 64, Hp, 2, Wp, 2).permute(0, 2, 4, 1, 3, 5).reshape(N, Hp, Wp, 64, 4)
    return win(v), win(S)


def conv1_pool(x, w, b):
    """(pooled output relu(max of the window) [N][Hp][Wp][64], the first arg-max of each window, v, S of conv1_windows)."""
    v, S = conv1_windows(x, w, b)
    best, arg = v.max(-1)               # torch.max returns the first maximal index on ties
    return torch.relu(best), arg, v, S


def window_patches(x):
    """The 3 x 3 pixel patch each conv position of each pool window reads: [N][Hp][Wp][4][9] (position py * 2 + px)."""
    N, H, W = x.shape
    Hp, Wp = H // 2, W // 2
    xp = F.pad(x, (1, 1, 1, 1))
    out = []
    for py in range(2):
        for px in range(2):
            taps = [xp[:, py + r:py + r + 2 * Hp:2, px + q:px + q + 2 * Wp:2] for r in range(3) for q in range(3)]
            out.append(torch.stack(taps, -1))
    return torch.stack(out, 3)


def conv1_dpre(code, dpool, H, W):
    """The pre-activation gradient the codes route: dpool at the winning conv position of each window when the ReLU bit (4) is
    set, 0 elsewhere.  code uint8 [N][Hp][Wp][64] (bit 1: py, bit 0: px), dpool [N][Hp][Wp][64]; returns [N][64][H][W]
    (the row / column an odd size leaves outside every window gets 0)."""
    N, Hp, Wp, C = dpool.shape
    c = code.long()
    g = torch.where((c & 4) != 0, dpool.double(), torch.zeros((), dtype=torch.float64, device=dpool.device))
    onehot = F.one_hot(c & 3, 4).double() * g[..., None]                       # [N][Hp][Wp][64][4]
    d = torch.zeros(N, C, H, W, dtype=torch.float64, device=dpool.device)
    d[:, :, :2 * Hp, :2 * Wp] = onehot.reshape(N, Hp, Wp, C, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(N, C, 2 * Hp, 2 * Wp)
    return d


def conv1_wgrad(x, code, dpool):
    """conv1's weight and bias gradient routed by the codes: (dw [64][9], S_w, db [64], S_b)."""
    N, H, W = x.shape
    d = conv1_dpre(code, dpool, H, W)
    dw = conv2d_weight(x[:, None], (64, 1, 3, 3), d, padding=1).reshape(64, 9)
    Sw = conv2d_weight(x.abs()[:, None], (64, 1, 3, 3), d.abs(), padding=1).reshape(64, 9)
    return dw, Sw, d.sum((0, 2, 3)), d.abs().sum((0, 2, 3))


# ------------------------------------------------------------------------------------------------------------------------
# 3 x 3 convolution (forward and data gradient) and its weight gradient
# ------------------------------------------------------------------------------------------------------------------------
def conv3x3(x, w, b=None, pad=1, relu=False, mask=None):
    """y = [relu](conv3x3(x, w, pad) + b) [* (mask > 0)], x [N][H][W][Cin], w [Cout][3][3][Cin]: (y, S) NHWC.  S includes |b|;
    where the mask is <= 0 both y and S are 0 (the kernel writes an exact 0 there)."""
    w4 = w.double().permute(0, 3, 1, 2).contiguous()
    bd = b.double() if b is not None else None
    y = _nhwc(F.conv2d(_nchw(x), w4, bd, padding=pad))
    S = _nhwc(F.conv2d(_nchw(x).abs(), w4.abs(), bd.abs() if bd is not None else None, padding=pad))
    if relu:
        y = torch.relu(y)
    if mask is not None:
        keep = (mask.double() > 0).double()
        y, S = y * keep, S * keep
    return y, S


def conv3x3_wgrad(x, dy, pad):
    """(dw [Cout][3][3][Cin], S_w, db [Cout], S_b) of y = conv3x3(x, w, pad) for the output gradient dy [N][Ho][Wo][Cout]."""
    Cin, Cout = x.shape[3], dy.shape[3]
    xd, dd = _nchw(x), _nchw(dy)
    dw = conv2d_weight(xd, (Cout, Cin, 3, 3), dd, padding=pad).permute(0, 2, 3, 1)
    Sw = conv2d_weight(xd.abs(), (Cout, Cin, 3, 3), dd.abs(), padding=pad).permute(0, 2, 3, 1)
    return dw, Sw, dd.sum((0, 2, 3)), dd.abs().sum((0, 2, 3))


def weight_flip(w):
    """lo_conv_weight_flip: [Cout][3][3][Cin] -> [Cin][3][3][Cout] with the taps reversed (the data gradient's weights)."""
    return w.flip(1, 2).permute(3, 1, 2, 0)


# ------------------------------------------------------------------------------------------------------------------------
# max-pool, ReLU mask, timing signal
# ------------------------------------------------------------------------------------------------------------------------
def _windows(y, kh, kw):
    N, H, W, C = y.shape
    Ho, Wo = H // kh, W // kw
    return y[:, :Ho * kh, :Wo * kw].double().reshape(N, Ho, kh, Wo, kw, C).permute(0, 1, 3, 5, 2, 4).reshape(N, Ho, Wo, C, kh * kw)


def maxpool(y, kh, kw):
    """Floor-mode max-pool of NHWC y with a (kh, kw) window and stride."""
    return _windows(y, kh, kw).amax(-1)


def maxpool_backward(y, dp, kh, kw):
    """dy routed to the FIRST maximum of each window in scan order (row-major, as nn.MaxPool2d), times (maximum > 0): the
    pooled input is a ReLU output, and relu'(0) = 0.  Rows and columns outside every window get 0."""
    N, H, W, C = y.shape
    Ho, Wo = H // kh, W // kw
    win = _windows(y, kh, kw)
    best, arg = win.max(-1)
    zero = torch.zeros((), dtype=torch.float64, device=dp.device)
    g = torch.where(best > 0, dp.double(), zero)
    route = torch.where(F.one_hot(arg, kh * kw) != 0, g[..., None], zero)      # +0 off the route, as the kernel writes
    dx = torch.zeros(N, H, W, C, dtype=torch.float64, device=dp.device)
    dx[:, :Ho * kh, :Wo * kw] = route.reshape(N, Ho, Wo, C, kh, kw).permute(0, 1, 4, 2, 5, 3).reshape(N, Ho * kh, Wo * kw, C)
    return dx


def relu_mask_cast(g, y):
    """lo_relu_mask_cast: g where y > 0, else 0."""
    return torch.where(y.double() > 0, g.double(), torch.zeros((), dtype=torch.float64, device=g.device))


def add_table(x, table):
    """lo_add_table: x + table, the [H][W][C] timing signal repeated per image."""
    return x.double() + table.double()[None]


# ------------------------------------------------------------------------------------------------------------------------
# the 'cnn' variant's strided conv as im2col + GEMMs
# ------------------------------------------------------------------------------------------------------------------------
def im2col(x, R, S_, stride, pad):
    """col [N*Ho*Wo][R*S*C] (tap-major columns) of NHWC x."""
    N, H, W, C = x.shape
    u = F.unfold(_nchw(x), (R, S_), padding=pad, stride=stride)             # [N][C*R*S][L], channel-major rows
    L_ = u.shape[-1]
    return u.view(N, C, R * S_, L_).permute(0, 3, 2, 1).reshape(N * L_, R * S_ * C)


def gemm_nt(a, b, bias=None, relu=False):
    """y = [relu](a b^T + bias), a [M][K], b [Nn][K]: (y, S)."""
    a, b = a.double(), b.double()
    y = a @ b.t()
    S = a.abs() @ b.abs().t()
    if bias is not None:
        y, S = y + bias.double(), S + bias.double().abs()
    return (torch.relu(y) if relu else y), S


def gemm_tn(a, b):
    """y = a^T b, a [M][Cout], b [M][K] (the strided conv's weight gradient dy^T col): (y, S)."""
    a, b = a.double(), b.double()
    return a.t() @ b, a.abs().t() @ b.abs()


def colsum(a):
    """Column sums of a [M][Nn] (the bias gradient): (sum, S)."""
    a = a.double()
    return a.sum(0), a.abs().sum(0)


def gemm_nn(a, b):
    """y = a b, a [M][Cout], b [Cout][K] (the strided conv's data gradient dcol = dy W): (y, S)."""
    a, b = a.double(), b.double()
    return a @ b, a.abs() @ b.abs()


def col2im(dcol, mask, N, H, W, C, R, S_, stride, pad):
    """dx [N][H][W][C]: the sum of the dcol entries of every window covering a pixel, times (mask > 0) if a mask is given:
    (dx, S)."""
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S_) // stride + 1

    def fold(v):
        u = v.double().view(N, Ho * Wo, R * S_, C).permute(0, 3, 2, 1).reshape(N, C * R * S_, Ho * Wo)
        return _nhwc(F.fold(u, (H, W), (R, S_), padding=pad, stride=stride))
    dx, S = fold(dcol), fold(dcol.abs())
    if mask is not None:
        keep = (mask.double() > 0).double()
        dx, S = dx * keep, S * keep
    return dx, S


# ------------------------------------------------------------------------------------------------------------------------
# the chain: EncoderCNN's launch order, forward and backward
# ------------------------------------------------------------------------------------------------------------------------
def chain(layers, p, img, denc, table=None, scale=1.0, offset=0.0):
    """EncoderCNN.forward_raw and backward_raw composed from the pieces above, in float64.  layers: EncoderCNN's layer tuples
    (latex_ocr_b200.encoder._LAYERS or _LAYERS_CNN); p: the kernels' parameter layouts ({"cnn.i.weight": [Cout][R][S][Cin],
    "cnn.i.bias": [Cout]}); img [N][1][H][W]; denc [N][H'][W'][512]; table: the timing signal [H'][W'][512] or None.
    Returns (encoder output, {acts}, {grads of the feature maps}, {parameter gradients in p's layouts})."""
    x = pixels(img, scale, offset)
    N, H, W = x.shape
    acts, grads, pg = {}, {}, {}
    P0, arg, v, _ = conv1_pool(x, p["cnn.0.weight"], p["cnn.0.bias"])
    best = v.max(-1).values
    code = (arg | torch.where(best > 0, 4, 0)).to(torch.uint8)
    acts["P0"] = P0
    cur = P0
    for l in layers[1:]:
        idx, cin, cout, pad, pool = l[:5]
        R, S_, stride = l[5] if len(l) > 5 else (3, 3, 1)
        w, b = p["cnn.%s.weight" % idx], p["cnn.%s.bias" % idx]
        if (R, S_, stride) == (3, 3, 1):
            y, _ = conv3x3(cur, w, b, pad, relu=True)
        else:
            col = im2col(cur, R, S_, stride, pad)
            acts["col" + idx] = col
            Ho, Wo = (cur.shape[1] + 2 * pad - R) // stride + 1, (cur.shape[2] + 2 * pad - S_) // stride + 1
            y = gemm_nt(col, w.reshape(cout, -1), b, relu=True)[0].view(N, Ho, Wo, cout)
        acts["Y" + idx] = cur = y
        if pool:
            acts["P" + idx] = cur = maxpool(y, *pool)
    out = add_table(cur, table) if table is not None else cur
    last = "Y" + layers[-1][0]
    grads[last] = relu_mask_cast(denc, acts[last])
    cfg = {l[0]: l for l in layers}
    for i in range(len(layers) - 1, 0, -1):
        l, prev = layers[i], layers[i - 1]
        idx, cin, cout, pad = l[:4]
        R, S_, stride = l[5] if len(l) > 5 else (3, 3, 1)
        xin = ("P" if prev[4] else "Y") + prev[0]
        xa, dy = acts[xin], grads["Y" + idx]
        mask = xa if xin.startswith("Y") else None
        if (R, S_, stride) == (3, 3, 1):
            dw, _, db, _ = conv3x3_wgrad(xa, dy, pad)
            grads[xin] = conv3x3(dy, weight_flip(p["cnn.%s.weight" % idx]), None, 2 - pad, mask=mask)[0]
        else:
            dy2 = dy.reshape(-1, cout)
            dw = gemm_tn(dy2, acts["col" + idx])[0].view(p["cnn.%s.weight" % idx].shape)
            db = colsum(dy2)[0]
            dcol = gemm_nn(dy2, p["cnn.%s.weight" % idx].reshape(cout, -1))[0]
            grads[xin] = col2im(dcol, mask, N, xa.shape[1], xa.shape[2], cin, R, S_, stride, pad)[0]
        pg["cnn.%s.weight" % idx], pg["cnn.%s.bias" % idx] = dw, db
        if xin.startswith("P") and xin != "P0":
            src = "Y" + xin[1:]
            grads[src] = maxpool_backward(acts[src], grads[xin], *cfg[xin[1:]][4])
    dw, _, db, _ = conv1_wgrad(x, code, grads["P0"])
    pg["cnn.0.weight"], pg["cnn.0.bias"] = dw.view(64, 3, 3, 1), db
    return out, acts, grads, pg
