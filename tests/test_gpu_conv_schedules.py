"""-m gpu: the encoder's tensor-core convolution and GEMM kernels (lo_tc.cu) under every schedule, and its bf16 / fp32
data-movement kernels (lo_conv.cu), element by element against float64.

The bound.  A convolution output is y = RN_bf16(sum_k x_k w_k (+ b)): the products of bf16 operands are exact in fp32, the
K = 9 Cin of them are summed in fp32 and the result is rounded once to bf16.  So against the float64 value ref of the same
bf16 operands every element must satisfy

    |y - ref| <= 0.5 ulp_bf16(ref) + 2^-16 (S + |b|),        S = sum_k |x_k| |w_k|   (float64, on |x| and |w|)

The first term is the one bf16 rounding (an exact value in [2^e, 2^(e+1)) rounds to within 2^(e-8)).  The second is the fp32
summation: a wgmma kernel updates its accumulator K/16 times (one k16 MMA each), the CUDA-core kernel K times (one FMA each);
every update errs by at most one fp32 rounding, 2^-24 of the running sum, whose magnitude is at most S.  Those errors have
random sign on sign-mixed data, so they add up to about sqrt(n) 2^-24 S with n <= K: at the largest K here (9 x 640 = 5760)
that is 76 x 2^-24 S < 2^-17.7 S.  2^-16 S is more than three times that, and still under half a bf16 ulp at typical
magnitudes, where |y| ~ S / sqrt(K) makes it at most 2^-16 sqrt(K) |y| < 2^-9.7 |y|, so a missed tap or a lost bias (of order
|y|) cannot hide in it.  ReLU is 1-Lipschitz, so a ReLU output follows the same bound; an output whose mask is <= 0 must be
exactly 0 (its bound is 0).

Worst |y - ref| / bound measured on an H100 80GB HBM3 (700 W power limit), over all shapes below:
    convolution, both schedules alike: 0.985 forward, 0.976 data gradient, 0.972 masked epilogue
    GEMM, conv_mc = 1 and 0 alike: 0.986 bf16 output, 0.041 fp32 output
The bf16 ratios approach 1 by construction: an exact value next to a bf16 rounding midpoint rounds with an error of nearly
half an ulp.  The fp32 GEMM outputs, where no bf16 rounding enters, show the accumulation alone: it used at most 4 % of its
allowance (at 8704 x 512 x 4096).

Every element written, nothing else: outputs are prefilled with NaN (an unwritten element fails the bound) inside a larger
buffer whose guard bands hold a sentinel that must survive the call.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

_SENTINEL = -1536.0                    # exact in bf16 and fp32, never produced by the data here
_ACC = 2.0 ** -16                      # fp32 accumulation allowance, relative to S (module docstring)


def _L():
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    assert L.lo_tc_available(), "the wgmma / TMA kernels need an sm_90 device"
    return _lib, L


def _guarded(shape, dtype, fill, guard):
    """(buffer, view): a tensor of `shape` filled with `fill`, inside a flat buffer with `guard` sentinel elements before and
    after it.  `guard` is a multiple of 64 elements, so the view keeps the buffer's 128-byte alignment."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((guard + n + guard,), _SENTINEL, dtype=dtype, device="cuda")
    view = buf[guard:guard + n].view(shape)
    view.fill_(fill)
    return buf, view


def _assert_guards(buf, guard, what):
    assert (buf[:guard] == _SENTINEL).all() and (buf[-guard:] == _SENTINEL).all(), "%s: wrote outside its output" % what


def _guard_for(row_elems):
    return max(4096, -(-row_elems // 64) * 64)


def _bits(t):
    """The bit patterns of a bf16 / fp32 tensor (bitwise comparisons: NaN never equals, -0 differs from +0)."""
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _half_ulp_bf16(ref):
    """Half the bf16 spacing at the float64 values `ref` (0 at 0): |ref| in [2^(e-1), 2^e) has spacing 2^(e-8)."""
    _, e = torch.frexp(ref)
    return torch.where(ref != 0, torch.ldexp(torch.full_like(ref, 0.5), e - 8), torch.zeros_like(ref))


def _check_bound(y, ref, bound, what):
    """Asserts |y - ref| <= bound element-wise (NaN fails) and returns the largest |y - ref| / bound."""
    d = (y.double() - ref).abs()
    ok = d <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s: %d of %d elements outside the bound; first at %s: got %r, float64 %r, bound %.3g"
                             % (what, bad.shape[0], y.numel(), i, y[i].item(), ref[i].item(), bound[i].item()))
    r = torch.where(bound > 0, d / bound.clamp_min(1e-300), torch.zeros_like(d))
    return r.max().item()


# ------------------------------------------------------------------------------------------------------------------------
# 3x3 convolution, every schedule
# ------------------------------------------------------------------------------------------------------------------------
def _conv_ref(x, w, pad):
    """float64 conv(x, w) and conv(|x|, |w|) of NHWC x [N][H][W][Cin] and w [Cout][3][3][Cin], both NHWC [N][Ho][Wo][Cout]:
    one image at a time, im2col (F.unfold) then a float64 matmul."""
    N, H, W, Cin = x.shape
    Cout = w.shape[0]
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    w2 = w.double().permute(0, 3, 1, 2).reshape(Cout, Cin * 9)          # (ci, r, s) order, as F.unfold lays out its rows
    wa = w2.abs()
    y = torch.empty(N, Ho * Wo, Cout, dtype=torch.float64, device="cuda")
    S = torch.empty_like(y)
    for n in range(N):
        cols = F.unfold(x[n:n + 1].double().permute(0, 3, 1, 2), 3, padding=pad)[0]
        y[n] = (w2 @ cols).t()
        S[n] = (wa @ cols.abs()).t()
    return y.view(N, Ho, Wo, Cout), S.view(N, Ho, Wo, Cout)


# (name, library options, impl): the persistent tensor-core kernel, then the CUDA-core kernel at bf16
_SCHEDULES = (("persistent", {}, 1),
              ("cuda_core", {}, 0))

# (N, H, W, Cin, Cout, pad) of a forward convolution.  The persistent kernel (132 SMs) runs min(tiles, 132) CTAs over CTA
# tiles of MT x 128 positions x NT channels (NT = 256 if Cout % 256 == 0, else 128 if Cout > 64, else 64; MT = 2 for NT <= 128,
# else 1); the position box is BW x BH = 128 with BW the smallest power of two >= Wo (8..128).  "dgrad" is the data
# gradient of the same layer: Cin and Cout swapped, pad' = 2 - pad.
_CONV_CASES = [
    # the encoder at the cfg2 geometry (B = 8, 128 x 512 images): the forward convs of layers 3, 6, 8, 11 and 14, each with its
    # data-gradient conv.  Several tiles per CTA on: fwd 3 (1024 M tiles, MT 2: 512 CTA tiles, 3.9 per SM), fwd 6 and fwd 8 (256
    # M tiles x 1 N tile of 256), fwd 11 (128 x 2 N tiles = 256), dgrad 3 (Cout 64, MT 2: 512) and dgrad 8 (256); one tile per
    # CTA on dgrad 6 (128), dgrad 11 (128), fwd 14 (56 x 2 = 112, Ho 14 in BH 2 boxes of 64) and dgrad 14 (64 x 2 = 128, pad 2)
    (8, 64, 256, 64, 128, 1),
    (8, 32, 128, 128, 256, 1),
    (8, 32, 128, 256, 256, 1),
    (8, 16, 128, 256, 512, 1),
    (8, 16, 64, 512, 512, 0),
    # odd M-tile count under MT 2 with more CTA tiles than SMs: 5 x 57 rows of one 128 box = 285 M tiles -> 143 CTA tiles, so
    # CTAs 0..10 run a second tile and the last pair holds one sub-tile (fwd NT 128 and dgrad NT 64 alike)
    (5, 57, 100, 64, 128, 1),
    # Cout 640 = five 128-wide N tiles: 5 does not divide 132, so a CTA's consecutive tiles (tile, tile + 132) use different
    # bias slices, and the double-buffered bias holds two different slices (64 M tiles, MT 2: 160 CTA tiles)
    (2, 32, 128, 64, 640, 1),
    # ragged channel tiles: Cout 200 = 128 + 72 (two N tiles, the second 72 wide: its 8-column groups past Cout are skipped;
    # Wo 40 in a 64 x 2 box: 30 M tiles in 15 pairs x 2 N tiles = 30 CTA tiles) and Cout 72 (one 128 tile, 56 columns past
    # Cout); their data gradients would have Cin 200 / 72, which the tensor-core kernel does not take (Cin % 64), so the second
    # use is the masked epilogue on the forward operands
    (3, 20, 40, 128, 200, 1),
    (2, 9, 13, 64, 72, 1),                     # Wo 13 in a 16 x 8 box, Ho 9 = 8 + 1
    # position boxes: Wo 6 <= 8 (8 x 16 box, Ho 40 = 2 x 16 + 8, 9 M tiles: odd under MT 2)
    (3, 40, 6, 64, 128, 1),
    # Wo 12 in 9..16 (16 x 8 box, Ho 11 = 8 + 3: the second box row holds 3 rows), pad 0; one N tile of 256, MT 1
    (2, 13, 14, 64, 256, 0),
    # Wo 140: two 128 x 1 boxes per row, the second 12 wide (116 positions of its sub-tile skipped); one N tile of 256, MT 1
    (2, 7, 140, 64, 256, 1),
    # the shapes of the former test_tc_conv3x3: Wo 128 (128 x 1), Wo 64 (64 x 2), Wo 62 / pad 0 (21 M tiles: odd), Wo 64 / pad 2,
    # Wo 30 in 17..32 (32 x 4 box, one CTA tile)
    (2, 8, 128, 64, 128, 1),
    (2, 16, 64, 128, 256, 1),
    (3, 16, 64, 512, 512, 0),
    (2, 14, 62, 512, 512, 2),
    (1, 6, 30, 256, 64, 1),
]


def _conv_uses(case):
    """The two uses of lo_conv3x3 at one shape: (name, x, w, bias, mask, relu, pad, ref, S), ref and S float64 NHWC."""
    _lib, L = _L()
    N, H, W, Cin, Cout, pad = case
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    g = torch.Generator(device="cuda").manual_seed(hash(case) & 0xffffffff)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / (3 * Cin ** 0.5)).bfloat16()
    b = 0.5 * torch.randn(Cout, device="cuda", generator=g)
    pre, S = _conv_ref(x, w, pad)
    bd = b.double()
    uses = [("fwd", x, w, b, None, 1, pad, torch.relu(pre + bd), S + bd.abs())]
    if Cout % 64 == 0:
        # data gradient: dx = conv(dy, flipped w, 2 - pad) * (mask > 0), mask = the ReLU output that fed the layer
        dy = torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g).bfloat16()
        wt = torch.empty(Cin, 3, 3, Cout, device="cuda", dtype=torch.bfloat16)
        _lib.check(L.lo_conv_weight_flip(_lib.ptr(w), _lib.ptr(wt), _lib.LO_BF16, Cin, Cout, _lib.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(_bits(wt), _bits(w.flip(1, 2).permute(3, 1, 2, 0)))
        mask = torch.relu(torch.randn(N, H, W, Cin, device="cuda", generator=g)).bfloat16()
        ref, Sd = _conv_ref(dy, wt, 2 - pad)
        keep = (mask > 0).double()
        uses.append(("dgrad", dy, wt, None, mask, 0, 2 - pad, ref * keep, Sd * keep))
    else:
        mask = torch.relu(torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g)).bfloat16()
        keep = (mask > 0).double()
        uses.append(("masked", x, w, None, mask, 0, pad, pre * keep, S * keep))
    return uses


def _run_conv(x, w, bias, mask, relu, pad, impl, opts):
    _lib, L = _L()
    N, H, W, Cin = x.shape
    Cout = w.shape[0]
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    guard = _guard_for(Wo * Cout)
    buf, y = _guarded((N, Ho, Wo, Cout), torch.bfloat16, float("nan"), guard)
    with _lib.option(**opts):
        _lib.check(L.lo_conv3x3(_lib.ptr(x), _lib.ptr(w), _lib.ptr(bias), _lib.ptr(mask), _lib.ptr(y), _lib.LO_BF16, N, H, W, Cin,
                                Cout, pad, relu, impl, _lib.stream_ptr()))
        torch.cuda.synchronize()
    return buf, guard, y


@pytest.mark.parametrize("N,H,W,Cin,Cout,pad", _CONV_CASES, ids=["x".join(map(str, c)) for c in _CONV_CASES])
def test_conv3x3_schedules(N, H, W, Cin, Cout, pad):
    """lo_conv3x3 at bf16, forward (bias + ReLU) and data gradient (flipped weights, ReLU mask), on the persistent tensor-core
    kernel and on the CUDA-core kernel: every element within the bound of the module docstring of the float64 value, nothing
    written outside the output."""
    for use, x, w, bias, mask, relu, pad_, ref, S in _conv_uses((N, H, W, Cin, Cout, pad)):
        bound = _half_ulp_bf16(ref) + _ACC * S
        for name, opts, impl in _SCHEDULES:
            what = "%s %s %s" % ("x".join(map(str, (N, H, W, Cin, Cout, pad))), use, name)
            buf, guard, y = _run_conv(x, w, bias, mask, relu, pad_, impl, opts)
            _assert_guards(buf, guard, what)
            ratio = _check_bound(y, ref, bound, what)
            print("%-40s worst |y - ref| / bound = %.4f" % (what, ratio))


# ------------------------------------------------------------------------------------------------------------------------
# tensor-core NT GEMM (tc_gemm_nt_ex) with and without the multicast A tile
# ------------------------------------------------------------------------------------------------------------------------
# (M, N, K, ldc): M > 64, so lo_gemm takes the 128 x 128 wgmma kernel, not the skinny one.  conv_mc = 1 pairs neighbouring N
# tiles in a cluster when cdiv(N, 128) is even.
_GEMM_CASES = [
    (300, 384, 512, 384),       # 3 N tiles (odd: no pairs), M = 2 x 128 + 44
    (1000, 200, 256, 216),      # 2 N tiles, the second 72 wide; ldc > N; M = 7 x 128 + 104
    (130, 512, 640, 520),       # 4 N tiles (two pairs), M = 128 + 2
    (777, 640, 128, 640),       # 5 N tiles (odd)
    (100, 512, 4096, 512),      # the cnn variant's im2col GEMM at its golden geometry (2 images x 5 x 10 positions, K = 2 x 4 x 512)
    (8704, 512, 4096, 512),     # ... and at the cfg2 geometry (8 images x 17 x 64 positions)
    (9600, 504, 512, 512),      # logits-sized: 4 N tiles, the last 120 wide, ldc > N
]


@pytest.mark.parametrize("M,N,K,ldc", _GEMM_CASES, ids=["x".join(map(str, c)) for c in _GEMM_CASES])
def test_tc_gemm_nt_multicast(M, N, K, ldc):
    """lo_gemm on tensor cores, C = A W^T: bf16 output with bias and ReLU, and fp32 output with bias accumulated onto C, under
    conv_mc = 1 and 0.  Bound of the module docstring (fp32: the accumulation term alone, with the old C as one more summand);
    the columns between N and ldc and the guard bands must keep their sentinel; both conv_mc values must agree bit for bit."""
    _lib, L = _L()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    Wt = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = 0.5 * torch.randn(N, device="cuda", generator=g)
    base = torch.randn(M, N, device="cuda", generator=g)
    P = A.double() @ Wt.double().t()
    S = A.double().abs() @ Wt.double().abs().t()
    bd = b.double()
    refs = {torch.bfloat16: torch.relu(P + bd), torch.float32: P + bd + base.double()}
    bounds = {torch.bfloat16: _half_ulp_bf16(refs[torch.bfloat16]) + _ACC * (S + bd.abs()),
              torch.float32: _ACC * (S + bd.abs() + base.double().abs())}
    del P, S
    guard = _guard_for(ldc)
    for dtype, acc, relu in ((torch.bfloat16, 0, 1), (torch.float32, 1, 0)):
        outs = {}
        for mc in (1, 0):
            what = "gemm %dx%dx%d ldc %d %s conv_mc=%d" % (M, N, K, ldc, str(dtype)[6:], mc)
            buf, C = _guarded((M, ldc), dtype, _SENTINEL, guard)
            C[:, :N] = base if acc else float("nan")
            with _lib.option(conv_mc=mc):
                _lib.check(L.lo_gemm(_lib.ptr(A), _lib.LO_BF16, _lib.ptr(Wt), _lib.LO_BF16, _lib.ptr(C), _lib.dt_of(C), M, N, K, K, 1, 1,
                                     K, ldc, 1, 0, 0, 0, _lib.ptr(b), acc, relu, _lib.LO_IMPL_TC, _lib.stream_ptr()))
                torch.cuda.synchronize()
            _assert_guards(buf, guard, what)
            assert (C[:, N:] == _SENTINEL).all(), "%s: wrote columns past N" % what
            ratio = _check_bound(C[:, :N], refs[dtype], bounds[dtype], what)
            print("%-50s worst |y - ref| / bound = %.4f" % (what, ratio))
            outs[mc] = _bits(C[:, :N])
        assert torch.equal(outs[0], outs[1]), "gemm %dx%dx%d %s: conv_mc = 1 and 0 differ bitwise" % (M, N, K, dtype)


# ------------------------------------------------------------------------------------------------------------------------
# the encoder's data-movement kernels: exact
# ------------------------------------------------------------------------------------------------------------------------
_DTYPES = [torch.float32, torch.bfloat16]


@pytest.mark.parametrize("dtype", _DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("k", [(2, 2), (2, 1), (1, 2)])
def test_maxpool_routes_ties_to_first_maximum(k, dtype):
    """lo_maxpool_forward / lo_maxpool_backward on ReLU-like inputs drawn from {0, 0.5, 1, 2}, so most windows have tied
    maxima: the forward takes the maximum, the backward routes dy to the FIRST maximum in scan order (row-major in the window,
    as nn.MaxPool2d) times (maximum > 0), and the rows and columns the floor mode drops (odd H and W) get 0.  Bitwise."""
    _lib, L = _L()
    kh, kw = k
    N, H, W, C = 2, 9, 11, 24
    Ho, Wo = H // kh, W // kw
    g = torch.Generator().manual_seed(kh * 10 + kw)
    vals = torch.tensor([0.0, 0.5, 1.0, 2.0])
    x = vals[torch.randint(0, 4, (N, H, W, C), generator=g)].to(dtype)
    dy = torch.randn(N, Ho, Wo, C, generator=g).to(dtype)
    # reference: windows unfolded to the last dimension in scan order; argmax returns the first maximum
    xw = x[:, :Ho * kh, :Wo * kw].double().reshape(N, Ho, kh, Wo, kw, C).permute(0, 1, 3, 5, 2, 4).reshape(N, Ho, Wo, C, kh * kw)
    y_ref = xw.amax(-1)
    win = F.one_hot(xw.argmax(-1), kh * kw).bool() & (y_ref > 0)[..., None]
    route = torch.where(win, dy.double()[..., None], 0.0)                  # +0 off the route, as the kernel writes
    dx_ref = torch.zeros(N, H, W, C, dtype=torch.float64)
    dx_ref[:, :Ho * kh, :Wo * kw] = route.reshape(N, Ho, Wo, C, kh, kw).permute(0, 1, 4, 2, 5, 3).reshape(N, Ho * kh, Wo * kw, C)
    st = _lib.stream_ptr()
    xc, dyc = x.cuda(), dy.cuda()
    guard = _guard_for(W * C)
    ybuf, y = _guarded((N, Ho, Wo, C), dtype, float("nan"), guard)
    _lib.check(L.lo_maxpool_forward(_lib.ptr(xc), _lib.ptr(y), _lib.dt_of(y), N, H, W, C, kh, kw, st))
    dxbuf, dx = _guarded((N, H, W, C), dtype, float("nan"), guard)
    _lib.check(L.lo_maxpool_backward(_lib.ptr(xc), _lib.ptr(y), _lib.ptr(dyc), _lib.ptr(dx), _lib.dt_of(dx), N, H, W, C, kh, kw, st))
    torch.cuda.synchronize()
    _assert_guards(ybuf, guard, "maxpool forward")
    _assert_guards(dxbuf, guard, "maxpool backward")
    assert torch.equal(_bits(y.cpu()), _bits(y_ref.to(dtype)))
    assert torch.equal(_bits(dx.cpu()), _bits(dx_ref.to(dtype)))


def _col_layout(unf, N, C, RS):
    """F.unfold's [N][C * R * S][L] (channel-major rows) -> the kernels' col [N * L][R * S * C] (tap-major)."""
    L_ = unf.shape[-1]
    return unf.view(N, C, RS, L_).permute(0, 3, 2, 1).reshape(N * L_, RS * C)


# (N, H, W, C, R, S, stride, pad)
_COL_CASES = [
    (2, 32, 128, 512, 2, 4, 2, 1),      # the cnn variant's Conv2d(512, 512, (2, 4), stride 2, padding 1) at the cfg2 geometry
    (3, 9, 13, 16, 2, 4, 2, 1),         # the same kernel on odd H and W with few channels
    (2, 11, 7, 8, 3, 3, 2, 1),          # overlapping windows: up to 4 of them cover a pixel
]


@pytest.mark.parametrize("dtype", _DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("N,H,W,C,R,S,stride,pad", _COL_CASES, ids=["x".join(map(str, c)) for c in _COL_CASES])
def test_im2col_col2im(N, H, W, C, R, S, stride, pad, dtype):
    """lo_im2col against F.unfold (bitwise: it only moves elements); lo_col2im, with and without the ReLU mask, against F.fold in
    float64.  col2im sums the n <= 4 windows covering a pixel in fp32 (at most n - 1 roundings of 2^-24 of sum |v| each, so
    2^-22 sum |v| allows for them) and bf16 rounds that once more (half a bf16 ulp)."""
    _lib, L = _L()
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
    K = R * S * C
    g = torch.Generator(device="cuda").manual_seed(H * 100 + W)
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    dcol = torch.randn(N * Ho * Wo, K, device="cuda", generator=g).to(dtype)
    mask = torch.relu(torch.randn(N, H, W, C, device="cuda", generator=g)).to(dtype)
    st = _lib.stream_ptr()
    dt = _lib.dt_of(x)
    guard = _guard_for(K)
    cbuf, col = _guarded((N * Ho * Wo, K), dtype, float("nan"), guard)
    _lib.check(L.lo_im2col(_lib.ptr(x), _lib.ptr(col), dt, N, H, W, C, R, S, stride, pad, st))
    torch.cuda.synchronize()
    _assert_guards(cbuf, guard, "im2col")
    ref = _col_layout(F.unfold(x.double().permute(0, 3, 1, 2), (R, S), padding=pad, stride=stride), N, C, R * S)
    assert torch.equal(_bits(col), _bits(ref.to(dtype)))

    def fold(v):
        u = v.double().view(N, Ho * Wo, R * S, C).permute(0, 3, 2, 1).reshape(N, C * R * S, Ho * Wo)
        return F.fold(u, (H, W), (R, S), padding=pad, stride=stride).permute(0, 2, 3, 1)

    dx_ref, dx_abs = fold(dcol), fold(dcol.abs())
    for m in (None, mask):
        keep = (m > 0).double() if m is not None else 1.0
        ref, Sa = dx_ref * keep, dx_abs * keep
        bound = 2.0 ** -22 * Sa + (_half_ulp_bf16(ref) if dtype == torch.bfloat16 else 0)
        xbuf, dx = _guarded((N, H, W, C), dtype, float("nan"), _guard_for(W * C))
        _lib.check(L.lo_col2im(_lib.ptr(dcol), _lib.ptr(m), _lib.ptr(dx), dt, N, H, W, C, R, S, stride, pad, st))
        torch.cuda.synchronize()
        what = "col2im %s" % ("masked" if m is not None else "")
        _assert_guards(xbuf, _guard_for(W * C), what)
        _check_bound(dx, ref, bound, what)


@pytest.mark.parametrize("dtype", _DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("K,N,ld_in,ld_out", [(100, 70, 80, 104), (512, 4096, 4096, 520)])
def test_transpose_with_padded_rows(K, N, ld_in, ld_out, dtype):
    """lo_transpose out[n][k] = in[k][n] with K and N not multiples of the 32 x 32 tile and padded rows on both sides (the
    second case is the cnn variant's weight transpose [512][4096] -> [4096][512]): bitwise, and the padding columns
    k >= K of the output and the guard bands keep their sentinel."""
    _lib, L = _L()
    g = torch.Generator(device="cuda").manual_seed(K + N)
    inp = torch.randn(K, ld_in, device="cuda", generator=g).to(dtype)
    guard = _guard_for(ld_out)
    buf, out = _guarded((N, ld_out), dtype, _SENTINEL, guard)
    out[:, :K] = float("nan")
    _lib.check(L.lo_transpose(_lib.ptr(inp), ld_in, _lib.ptr(out), ld_out, _lib.dt_of(inp), K, N, _lib.stream_ptr()))
    torch.cuda.synchronize()
    _assert_guards(buf, guard, "transpose")
    assert (out[:, K:] == _SENTINEL).all(), "transpose wrote the padding columns"
    assert torch.equal(_bits(out[:, :K]), _bits(inp[:, :N].t()))


@pytest.mark.parametrize("dtype", _DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("N,H,W,C", [(3, 5, 7, 24), (8, 14, 62, 512)])
def test_add_table(N, H, W, C, dtype):
    """lo_add_table out = y + table (the timing signal, fp32 [H][W][C], repeated per image): fp32 arithmetic, then one cast to
    the storage type, bitwise."""
    _lib, L = _L()
    g = torch.Generator(device="cuda").manual_seed(N * H * W)
    y = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    table = torch.randn(H, W, C, device="cuda", generator=g)
    guard = _guard_for(W * C)
    buf, out = _guarded((N, H, W, C), dtype, float("nan"), guard)
    _lib.check(L.lo_add_table(_lib.ptr(y), _lib.ptr(table), _lib.ptr(out), _lib.dt_of(y), N, H * W * C, _lib.stream_ptr()))
    torch.cuda.synchronize()
    _assert_guards(buf, guard, "add_table")
    assert torch.equal(_bits(out), _bits((y.float() + table).to(dtype)))


@pytest.mark.parametrize("dtype", _DTYPES, ids=["fp32", "bf16"])
def test_relu_mask_cast(dtype):
    """lo_relu_mask_cast out = g * (y > 0) cast to the storage type, with y holding exact zeros, -0 and negatives: bitwise."""
    _lib, L = _L()
    n = 8 * 12345
    g = torch.Generator(device="cuda").manual_seed(9)
    grad = torch.randn(n, device="cuda", generator=g)
    y = torch.relu(torch.randn(n, device="cuda", generator=g)).to(dtype)
    y[::7] = -0.0
    y[3::11] = -1.0
    guard = _guard_for(64)
    buf, out = _guarded((n,), dtype, float("nan"), guard)
    _lib.check(L.lo_relu_mask_cast(_lib.ptr(grad), _lib.ptr(y), _lib.ptr(out), _lib.dt_of(y), n, _lib.stream_ptr()))
    torch.cuda.synchronize()
    _assert_guards(buf, guard, "relu_mask_cast")
    assert torch.equal(_bits(out), _bits(torch.where(y.float() > 0, grad, torch.zeros_like(grad)).to(dtype)))
