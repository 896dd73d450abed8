"""-m gpu: the encoder (EncoderCNN.forward_raw / backward_raw) launch by launch against float64, as it runs: the kernels chained
through the workspace, with the arg-max / ReLU codes, masks and buffers handed from one launch to the next, under every
schedule of its convolutions and in both precisions.

Each case fills every activation and gradient buffer of the workspace, the weight-flip buffers, the im2col buffer and the whole
gradient store with a finite sentinel (conv1's code buffer with 0xff: valid codes are 0..7), runs forward_raw(img,
need_grad=True) and backward_raw with a random d enc, and then rebuilds every launch's output in float64
(tests/encoder_step_ref.py) from the buffers that launch read: the bf16 shadows of the 3 x 3 and strided weights where the
kernels read them (fp32 masters in fp32 mode), the fp32 masters of conv1 and of the biases, the previous launch's stored output,
conv1's own codes.  So an error never compounds from launch to launch.

Bounds.  A sum y of n terms evaluated in fp32 errs by at most d u S to first order, u = 2^-24, S the float64 sum of the
magnitudes of its terms and d the longest chain of fp32 additions one term passes through (its thread's FMA chain, then any
warp tree, cluster sum or atomics after it).  Those roundings have random sign on these sign-mixed terms and grow like
sqrt(d); every check here allows

    |y - ref| <= A(d) S (+ half a bf16 ulp of ref where y is stored in bf16),     A(d) = u max(256, 4 sqrt(d)),

that is 2^-16 S up to d = 4096 (the rule of tests/test_gpu_conv_schedules.py) and four times the sqrt(d) u S scale above.
The chain lengths d of each kernel, as its launcher sizes it:
  * convolutions (tensor cores and CUDA cores, forward and data gradient) and the strided conv's NT GEMM: K = 9 Cin (or
    R S C), the CUDA-core kernel one FMA per term, the wgmma kernels one k16 MMA per 16 terms: d <= K + 1 (the bias).
  * conv3x3_wgrad_kernel (CUDA cores): splits = min(cdiv(528, 9 cdiv(Cin, 64) cdiv(Cout, 64)), cdiv(P, 512)), at most 2 under
    "deterministic"; each thread runs one FMA chain over its split's P / splits positions, the splits meet in atomics:
    d = cdiv(P, splits) + splits.  At B = 8, 128 x 512: cnn.3 30 splits of 4,384 positions; cnn.14 one chain of 6,944.
  * tc_wgrad_kernel: one k16 MMA per 16 positions of a split, then at most P / 64 splits (atomics), or 8 under
    "deterministic" (an ordered cluster sum): d <= P / 16 + P / 64.  At the bench shape cnn.3 has P = 1,048,576.
  * conv1_pool_wgrad_code_kernel: grid = min(cdiv(npos, 32), 528) blocks, each lane one FMA chain over npos / (32 grid)
    pooled positions, then a 5-level warp tree and the grid partials (atomics, or the ordered block sum):
    d = cdiv(npos, 32 grid) + 5 + grid; npos = N H/2 W/2 (596 at the bench shape).
  * column sums (the bias gradients) and the strided conv's TN weight GEMM: d <= M, the number of rows.
  * col2im: at most 2 windows of the (2, 4) stride-2 conv cover a pixel: 2^-22 S.
Every conv output is rounded once to its storage type; ReLU and the mask are 1-Lipschitz, and a masked element must be exactly 0.

conv1's codes.  The window values v_i of a pooled output carry the bound e_i = 2^-16 S_i (nine FMAs and the bias).  The code
must name a position whose float64 value lies within e_chosen + e_max of the window's maximum; where two positions read
identical 3 x 3 pixel patches (exact ties, as in flat white regions), the earlier one must win; the ReLU bit must be set where
the maximum exceeds the window's largest e_i and clear where it is below minus that.  P0 is relu of the chosen value.

Exact, bit for bit: max-pool forward and backward (first maximum in scan order, times maximum > 0, zeros outside every window)
on the kernel's own inputs; relu_mask_cast; add_table (fp32 add, one cast); im2col; the weight flip and the strided conv's
weight transpose; the no-grad forward (lo_conv1_pool_forward, _u8 or _norm, as decoding runs it) against the training forward;
and, under "deterministic", the recomputing conv1 weight-gradient kernels (lo_conv1_pool_wgrad, _u8, _norm) against the
code kernel: the same non-zero FMAs in the same order, and the same block partials.

Every element written: no buffer keeps the sentinel (the rows and columns an odd size leaves outside a pool window are
checked to be exactly 0 by the max-pool backward), every code is below 8, and the gradient store's alignment padding, which
no kernel owns, keeps it.  Under "deterministic" two runs agree bit for bit in every buffer.

Worst |y - ref| / bound per quantity over every case and schedule, measured on an H100 80GB HBM3 (700 W power limit); the
whole file (31 tests) ran in 14 s there:
                            fp32 storage    bf16 storage
    conv1 arg-max value         0.0000          0.0003
    P0                          0.012           0.996
    conv forward                0.022           0.982
    conv data gradient          0.027           0.993
    dcol                        0.021           0.987
    col2im                      0.250           1.000
    conv dw                     0.033           0.100
    conv db                     0.007           0.002
    conv1 dw                    0.014           0.008
    conv1 db                    0.005           0.002
The bf16 ratios approach 1 by construction: an exact value next to a rounding midpoint rounds with nearly half an ulp.  The
fp32 ones show the accumulation alone; the largest share of an allowance used by a weight gradient was 10 %, on the
tensor-core kernel at the bench shape.  Case b8's formula images hold 598,616 pairs of window positions with identical patches.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import encoder_step_ref as es
from step_check import ACC, SENTINEL, Checker, half_ulp_bf16

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
CODE_SENTINEL = 0xff


def allow(d):
    """The relative allowance A(d) of an fp32 sum whose longest chain has d roundings (module docstring)."""
    return U * max(256.0, 4.0 * math.sqrt(d))


def cdiv(a, b):
    return -(-a // b)


def wgrad_depth(tc, P, Cin, Cout, det):
    """d of lo_conv3x3_wgrad's weight gradient (module docstring)."""
    if tc and Cin % 64 == 0 and Cout % 128 == 0:
        return P // 16 + cdiv(P, 64)
    splits = max(1, min(cdiv(528, 9 * cdiv(Cin, 64) * cdiv(Cout, 64)), cdiv(P, 512), 2 if det else 1 << 30))
    return cdiv(cdiv(P, splits), 16) * 16 + splits


def conv1_wgrad_depth(npos):
    grid = min(cdiv(npos, 32), 528)
    return cdiv(npos, 32 * grid) + 5 + grid


class _Cfg:
    def __init__(self, variant, positional, norm):
        self.encoder_cnn = variant
        self.positional_embeddings = positional
        self.input_norm = norm


def formula_images(N, H, W, g):
    """Formula-like pixels on the GPU: 255 background, dark horizontal and vertical strokes on a few percent of the pixels,
    the last image all white."""
    def strokes(p, k):
        seed = (torch.rand(N, 1, H, W, device="cuda", generator=g) < p).float()
        return F.max_pool2d(seed, k, stride=1, padding=(k[0] // 2, k[1] // 2))
    ink = torch.maximum(strokes(0.004, (1, 9)), strokes(0.003, (9, 1))) > 0
    dark = torch.randint(0, 120, (N, 1, H, W), device="cuda", generator=g).float()
    img = torch.where(ink, dark, torch.full_like(dark, 255.0))
    img[-1] = 255.0
    return img


# name: (variant, N, H, W, pixels, input dtype, input_norm, positional embeddings)
_CASES = {
    "b8": ("vanilla", 8, 128, 512, "formula", torch.float32, None, True),
    "bench": ("vanilla", 64, 128, 512, "formula", torch.float32, None, True),
    # 39 = 8 * 4 + 7 and 143 = 8 * 17 + 7: conv1's pool drops a row and a column, cnn.3's pool too (19 x 71), cnn.8's (2, 1)
    # pool a row (9 -> 4), cnn.11's (1, 2) pool a column (35 -> 17)
    "odd": ("vanilla", 3, 39, 143, "formula", torch.float32, None, True),
    "u8": ("vanilla", 2, 64, 256, "formula", torch.uint8, None, True),
    "tf": ("vanilla", 2, 64, 256, "formula", torch.float32, "tf", True),
    "tf_u8": ("vanilla", 2, 64, 256, "formula", torch.uint8, "tf", True),
    "nopos": ("vanilla", 2, 64, 256, "formula", torch.float32, None, False),
    "cnn": ("cnn", 4, 64, 256, "formula", torch.float32, None, True),
    "rand": ("vanilla", 2, 64, 256, "random", torch.float32, None, True),
}
_SMALL = ["u8", "tf", "tf_u8", "nopos", "rand"]

# name: (precision, conv_impl, library options, cases)
_SCHEDULES = {
    "fp32_simt": ("fp32", "simt", {}, ["b8", "odd", "cnn"] + _SMALL),
    "bf16_simt": ("bf16", "simt", {}, ["b8", "odd", "cnn", "u8"]),
    "tc": ("bf16", "tc", {}, ["b8", "bench", "odd", "cnn"] + _SMALL),
    "wgrad256": ("bf16", "tc", {"wgrad256": 1}, ["b8", "cnn"]),
    "det_tc": ("bf16", "tc", {"deterministic": 1}, ["b8", "bench", "odd", "cnn"]),
    "det_fp32": ("fp32", "simt", {"deterministic": 1}, ["b8", "odd", "cnn"]),
}
_PARAMS = [(s, c) for s, v in _SCHEDULES.items() for c in v[3]]

_WORST = {}


def _lib():
    from latex_ocr_b200 import _lib as lib
    return lib


def _buffers(ws):
    """Every buffer of the workspace the encoder writes, by name (activations, gradients, weight flips, im2col, output)."""
    out = {}
    for k, t in ws["acts"].items():
        out["act " + k] = t
    for k, t in (ws["grads"] or {}).items():
        out["grad " + k] = t
    for k, t in ws["wflip"].items():
        out["wflip " + k] = t
    for k, t in ws.items():
        if k.startswith("col"):
            out[k] = t
    out["out"] = ws["out"]
    return out


def _prefill(enc, ws):
    for t in _buffers(ws).values():
        t.fill_(SENTINEL)
    ws["code0"] = torch.full(ws["acts"]["P0"].shape, CODE_SENTINEL, dtype=torch.uint8, device="cuda")
    enc.store.grad.fill_(SENTINEL)


def _run(enc, img, denc, opts):
    """One forward_raw(need_grad=True) + backward_raw from sentinel-filled buffers.  Returns (ws, snapshots of the buffers
    the backward overwrites or that a later call would: col after the forward, the output)."""
    lib = _lib()
    N, _, H, W = img.shape
    ws = enc._workspace(N, H, W, True)
    _prefill(enc, ws)
    with lib.option(**opts):
        out = enc.forward_raw(img, need_grad=True)
        snap = {k: t.clone() for k, t in ws.items() if k.startswith("col")}
        snap["out"] = out.clone()
        enc.backward_raw(img.shape, denc)
        torch.cuda.synchronize()
    return ws, snap


def _state(enc, ws):
    d = {k: t.clone() for k, t in _buffers(ws).items()}
    d["code0"] = ws["code0"].clone()
    d["store.grad"] = enc.store.grad.clone()
    return d


def _check_written(enc, ws, positional):
    for k, t in _buffers(ws).items():
        if k == "out" and not positional:
            continue
        assert not bool((t == SENTINEL).any()), "%s keeps the sentinel in %d elements" % (k, int((t == SENTINEL).sum()))
    assert bool((ws["code0"] < 8).all()), "conv1 left %d codes unwritten" % int((ws["code0"] >= 8).sum())
    S = enc.store
    owned = torch.zeros(S.numel, dtype=torch.bool, device="cuda")
    for name, (off, n, _) in S.offsets.items():
        assert not bool((S.grad[off:off + n] == SENTINEL).any()), "gradient %s not written everywhere" % name
        owned[off:off + n] = True
    assert bool((S.grad[~owned] == SENTINEL).all()), "a kernel wrote the gradient store's padding"


def _check_conv1(ck, enc, ws, img, sc, of, dt, opts):
    lib = _lib()
    L = lib.lib()
    A, G, S = ws["acts"], ws["grads"], enc.store
    bf = dt == torch.bfloat16
    x = es.pixels(img, sc, of)
    _, vmax_arg, v, Sv = es.conv1_pool(x, S.f32("cnn.0.weight"), S.f32("cnn.0.bias"))
    e = ACC * Sv
    code = ws["code0"].long()
    chosen, relu_bit = code & 3, (code & 4) != 0
    v_ch = v.gather(-1, chosen[..., None])[..., 0]
    e_ch = e.gather(-1, chosen[..., None])[..., 0]
    vmax = v.max(-1).values
    e_max = e.gather(-1, vmax_arg[..., None])[..., 0]
    ck.bound("conv1 arg-max value", v_ch, vmax, e_ch + e_max)
    # exact ties: a later position whose 3 x 3 patch equals an earlier one's must never be chosen
    patches = es.window_patches(x)
    ties = 0
    for j in range(1, 4):
        for i in range(j):
            same = (patches[..., i, :] == patches[..., j, :]).all(-1)[..., None]
            bad = (chosen == j) & same
            assert not bool(bad.any()), "conv1: %d codes choose position %d over the identical earlier position %d" % (
                int(bad.sum()), j, i)
            ties += int(same.sum())
    e_w = e.amax(-1)
    assert not bool((~relu_bit & (vmax > e_w)).any()), "conv1: ReLU bit clear on a positive maximum"
    assert not bool((relu_bit & (vmax < -e_w)).any()), "conv1: ReLU bit set on a negative maximum"
    ref = torch.relu(v_ch)
    ck.bound("P0", A["P0"], ref, e_ch + (half_ulp_bf16(ref) if bf else 0))
    assert bool((A["P0"][~relu_bit] == 0).all()) and bool((A["P0"][relu_bit] > 0).all()), "P0 disagrees with its ReLU bits"

    # weight and bias gradient of the code kernel, routed by its own codes
    N, _, H, W = img.shape
    dw, Sw, db, Sb = es.conv1_wgrad(x, ws["code0"], G["P0"])
    a = allow(conv1_wgrad_depth(N * (H // 2) * (W // 2)))
    ck.bound("conv1 dw", S.g("cnn.0.weight").view(64, 9), dw, a * Sw)
    ck.bound("conv1 db", S.g("cnn.0.bias"), db, a * Sb)
    # the recomputing kernels on the same dpool
    u8 = img.dtype == torch.uint8
    rw = torch.full((64, 9), SENTINEL, device="cuda")
    rb = torch.full((64,), SENTINEL, device="cuda")
    st, dtc = lib.stream_ptr(), lib.dt_of(G["P0"])
    with lib.option(**opts):
        if enc.input_norm == "tf":
            lib.check(L.lo_conv1_pool_wgrad_norm(lib.ptr(img), int(u8), sc, of, lib.ptr(S.f32("cnn.0.weight")), lib.ptr(S.f32("cnn.0.bias")),
                                                 lib.ptr(G["P0"]), dtc, lib.ptr(rw), lib.ptr(rb), N, H, W, st))
        else:
            fn = L.lo_conv1_pool_wgrad_u8 if u8 else L.lo_conv1_pool_wgrad
            lib.check(fn(lib.ptr(img), lib.ptr(S.f32("cnn.0.weight")), lib.ptr(S.f32("cnn.0.bias")), lib.ptr(G["P0"]), dtc,
                         lib.ptr(rw), lib.ptr(rb), N, H, W, st))
        torch.cuda.synchronize()
    ck.bound("conv1 dw", rw, dw, a * Sw)
    ck.bound("conv1 db", rb, db, a * Sb)
    if opts.get("deterministic"):
        ck.exact("conv1 recompute dw", rw, S.g("cnn.0.weight").view(64, 9))
        ck.exact("conv1 recompute db", rb, S.g("cnn.0.bias"))
    return ties


def _check_flow(ck, enc, ws, snap, img, denc, opts):
    """Every launch of forward_raw / backward_raw from the buffers it read."""
    A, G, S = ws["acts"], ws["grads"], enc.store
    dt = enc.tdtype
    bf = dt == torch.bfloat16
    tc = enc._impl() == _lib().LO_IMPL_TC
    det = bool(opts.get("deterministic"))

    def rnd(ref):
        return half_ulp_bf16(ref) if bf else 0.0

    layers = enc.layers
    # forward
    x = A["P0"]
    for l in layers[1:]:
        idx, cin, cout, pad, pool = l[:5]
        R, S_, stride = l[5] if len(l) > 5 else (3, 3, 1)
        w, b = S.w("cnn.%s.weight" % idx), S.f32("cnn.%s.bias" % idx)
        if (R, S_, stride) == (3, 3, 1):
            ref, Sy = es.conv3x3(x, w, b, pad, relu=True)
            d = 9 * cin + 1
        else:
            col = snap["col" + idx]
            ck.exact("im2col", col, es.im2col(x, R, S_, stride, pad))
            ref, Sy = es.gemm_nt(col, w.reshape(cout, -1), b, relu=True)
            ref, Sy = ref.view(A["Y" + idx].shape), Sy.view(A["Y" + idx].shape)
            d = R * S_ * cin + 1
        y = A["Y" + idx]
        ck.bound("conv forward", y, ref, rnd(ref) + allow(d) * Sy)
        x = y
        if pool:
            ck.exact("maxpool forward", A["P" + idx], es.maxpool(y, *pool))
            x = A["P" + idx]
    if enc._config.positional_embeddings:
        ck.exact("add_table", snap["out"], (x.float() + ws["table"]).to(dt))
    # backward
    last = "Y" + layers[-1][0]
    ck.exact("relu_mask_cast", G[last], es.relu_mask_cast(denc, A[last]))
    cfg = {l[0]: l for l in layers}
    for i in range(len(layers) - 1, 0, -1):
        l, prev = layers[i], layers[i - 1]
        idx, cin, cout, pad = l[:4]
        R, S_, stride = l[5] if len(l) > 5 else (3, 3, 1)
        xin = ("P" if prev[4] else "Y") + prev[0]
        xa, dy = A[xin], G["Y" + idx]
        mask = xa if xin.startswith("Y") else None
        w = S.w("cnn.%s.weight" % idx)
        if (R, S_, stride) == (3, 3, 1):
            wt = ws["wflip"][idx].view(cin, 3, 3, cout)
            ck.exact("weight flip", wt, es.weight_flip(w))
            dw, Sw, db, Sb = es.conv3x3_wgrad(xa, dy, pad)
            P = dy.shape[0] * dy.shape[1] * dy.shape[2]
            ck.bound("conv dw", S.g("cnn.%s.weight" % idx), dw, allow(wgrad_depth(tc, P, cin, cout, det)) * Sw)
            ck.bound("conv db", S.g("cnn.%s.bias" % idx), db, allow(P) * Sb)
            ref, Sd = es.conv3x3(dy, wt, None, 2 - pad, mask=mask)
            ck.bound("conv data gradient", G[xin], ref, rnd(ref) + allow(9 * cout) * Sd)
        else:
            K = R * S_ * cin
            ck.exact("weight transpose", ws["wflip"][idx].view(K, cout), w.reshape(cout, K).t())
            dy2 = dy.reshape(-1, cout)
            M = dy2.shape[0]
            dw, Sw = es.gemm_tn(dy2, snap["col" + idx])
            ck.bound("conv dw", S.g("cnn.%s.weight" % idx).reshape(cout, K), dw, allow(M) * Sw)
            db, Sb = es.colsum(dy2)
            ck.bound("conv db", S.g("cnn.%s.bias" % idx), db, allow(M) * Sb)
            dcol = ws["col" + idx]                      # the data-gradient GEMM writes dcol over col
            ref, Sd = es.gemm_nn(dy2, w.reshape(cout, K))
            ck.bound("dcol", dcol, ref, rnd(ref) + allow(cout) * Sd)
            N_, H_, W_ = xa.shape[:3]
            ref, Sd = es.col2im(dcol, mask, N_, H_, W_, cin, R, S_, stride, pad)
            ck.bound("col2im", G[xin], ref, rnd(ref) + 2.0 ** -22 * Sd)
        if xin.startswith("P") and xin != "P0":
            src = "Y" + xin[1:]
            ck.exact("maxpool backward", G[src], es.maxpool_backward(A[src], G[xin], *cfg[xin[1:]][4]))


@pytest.mark.parametrize("schedule,case", _PARAMS, ids=["%s-%s" % p for p in _PARAMS])
def test_encoder_launches_against_float64(schedule, case):
    from latex_ocr_b200.encoder import EncoderCNN
    lib = _lib()
    precision, impl, opts, _ = _SCHEDULES[schedule]
    variant, N, H, W, kind, in_dt, norm, positional = _CASES[case]
    g = torch.Generator(device="cuda").manual_seed(11 + list(_CASES).index(case))
    torch.manual_seed(17)
    enc = EncoderCNN(_Cfg(variant, positional, norm), device="cuda", precision=precision, impl=impl)
    if kind == "formula":
        img = formula_images(N, H, W, g)
    else:
        img = torch.rand(N, 1, H, W, device="cuda", generator=g) * 255.0
    img = img.to(in_dt)
    Ho, Wo = enc.out_hw(H, W)
    denc = torch.randn(N, Ho, Wo, 512, device="cuda", generator=g)
    sc, of = (1.0 / 128.0, -1.0) if norm == "tf" else (1.0, 0.0)
    ck = Checker("%s %s" % (schedule, case))

    ws, snap = _run(enc, img, denc, opts)
    _check_written(enc, ws, positional)
    first = _state(enc, ws) if opts.get("deterministic") else None
    ties = _check_conv1(ck, enc, ws, img, sc, of, enc.tdtype, opts)
    if kind == "formula":
        assert ties > 0, "formula images without exactly tied windows"
    _check_flow(ck, enc, ws, snap, img, denc, opts)

    # the no-grad forward (lo_conv1_pool_forward / _u8 / _norm, as decoding runs it) computes the same encoder bit for bit
    acts = {k: t.clone() for k, t in ws["acts"].items()}
    with lib.option(**opts):
        out = enc.forward_raw(img, need_grad=False)
        torch.cuda.synchronize()
    for k, t in acts.items():
        ck.exact("no-grad forward " + k, ws["acts"][k], t)
    ck.exact("no-grad forward output", out, snap["out"])

    if first is not None:
        _run(enc, img, denc, opts)
        again = _state(enc, ws)
        for k, t in first.items():
            assert torch.equal(t.view(torch.uint8), again[k].view(torch.uint8)), \
                "%s %s: two deterministic runs differ in %s" % (schedule, case, k)

    for k, r in ck.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), r)
    print("\n[%s %s] exact ties in conv1 windows: %d" % (schedule, case, ties))
    for k in sorted(ck.worst):
        if not k.startswith("no-grad") and ck.worst[k] > 0:
            print("  %-24s worst |y - ref| / bound = %.4f" % (k, ck.worst[k]))


def test_cuda_core_conv_beyond_65535_position_tiles():
    """lo_conv3x3 on CUDA cores with more than 65,535 tiles of 64 output positions (2 x 1026 x 2048 = 4,202,496 positions,
    past 65,535 x 64 = 4,194,240): it launches, writes every element, and the last image's last rows, the ones the old grid
    would have put past its limit, match float64."""
    lib = _lib()
    L = lib.lib()
    N, H, W, Cin, Cout = 2, 1026, 2048, 16, 8
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / 12.0
    b = torch.randn(Cout, device="cuda", generator=g)
    y = torch.full((N, H, W, Cout), float("nan"), device="cuda")
    lib.check(L.lo_conv3x3(lib.ptr(x), lib.ptr(w), lib.ptr(b), None, lib.ptr(y), lib.LO_F32, N, H, W, Cin, Cout, 1, 1,
                           lib.LO_IMPL_SIMT, lib.stream_ptr()))
    torch.cuda.synchronize()
    assert not bool(y.isnan().any()), "%d outputs not written" % int(y.isnan().sum())
    ref, S = es.conv3x3(x[-1:, -9:], w, b, 1, relu=True)          # rows H-9..H-1; the first one sees a false zero pad
    ck = Checker("conv3x3 %dx%dx%dx%d" % (N, H, W, Cin))
    ck.bound("last rows", y[-1:, -8:], ref[:, 1:], allow(9 * Cin + 1) * S[:, 1:])
