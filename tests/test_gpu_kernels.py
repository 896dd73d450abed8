"""-m gpu: per-kernel numerics of the C-ABI entry points against plain PyTorch fp32 ops of the same
operation (the op-level reference) — the end-to-end parity against the oracle is in test_gpu_parity.py."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from util import relerr

pytestmark = pytest.mark.gpu


def _L():
    from latex_ocr_b200 import _lib
    return _lib, _lib.lib()


def _gemm(A, B, C, M, N, K, sam, sak, sbk, sbn, ldc, batch=1, sA=0, sB=0, sC=0, bias=None, acc=0, relu=0, impl=0):
    _lib, L = _L()
    _lib.check(L.lo_gemm(_lib.ptr(A), _lib.dt_of(A), _lib.ptr(B), _lib.dt_of(B), _lib.ptr(C), _lib.dt_of(C), M, N, K,
                         sam, sak, sbk, sbn, ldc, batch, sA, sB, sC, _lib.ptr(bias), acc, relu, impl, _lib.stream_ptr()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N,K", [(64, 3072, 512), (100, 70, 33), (868, 512, 512), (5, 8, 4096), (1, 500, 512)])
def test_gemm_nt_fp32(M, N, K):
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda")
    b = torch.randn(N, device="cuda")
    C = torch.zeros(M, N, device="cuda")
    _gemm(A, W, C, M, N, K, K, 1, 1, K, N, bias=b)
    ref = (A.double() @ W.double().t() + b.double()).float()
    assert relerr(C, ref) < 2e-6
    C2 = torch.ones(M, N, device="cuda")
    _gemm(A, W, C2, M, N, K, K, 1, 1, K, N, acc=1)
    assert relerr(C2, (A.double() @ W.double().t() + 1).float()) < 2e-5   # split-K atomics for long K


def test_gemm_relu_and_dtypes():
    torch.manual_seed(1)
    M, N, K = 130, 96, 256
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda")
    Ab, Wb = A.bfloat16(), W.bfloat16()
    ref = torch.relu(Ab.double() @ Wb.double().t()).float()
    C = torch.zeros(M, N, device="cuda")
    _gemm(Ab, Wb, C, M, N, K, K, 1, 1, K, N, relu=1)
    assert relerr(C, ref) < 1e-5
    Cb = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    _gemm(Ab, Wb, Cb, M, N, K, K, 1, 1, K, N, relu=1)
    assert relerr(Cb.float(), ref) < 1e-2
    C3 = torch.zeros(M, N, device="cuda")
    _gemm(A, Wb, C3, M, N, K, K, 1, 1, K, N)
    assert relerr(C3, (A.double() @ Wb.double().t()).float()) < 1e-5


def test_gemm_tn_nn_batched():
    torch.manual_seed(2)
    Kd, M, N = 3000, 96, 40
    A = torch.randn(Kd, M, device="cuda")
    B = torch.randn(Kd, N, device="cuda")
    C = torch.zeros(M, N, device="cuda")
    _gemm(A, B, C, M, N, Kd, 1, M, N, 1, N)                       # A^T B  (split-K path)
    assert relerr(C, (A.double().t() @ B.double()).float()) < 1e-5
    A2 = torch.randn(50, 64, device="cuda")
    B2 = torch.randn(64, 72, device="cuda")
    C2 = torch.zeros(50, 80, device="cuda")                      # ldc > N
    _gemm(A2, B2, C2, 50, 72, 64, 64, 1, 72, 1, 80)
    assert relerr(C2[:, :72], (A2.double() @ B2.double()).float()) < 1e-5
    assert C2[:, 72:].abs().max().item() == 0
    # batched, strided like denc += alphas^T dctx
    Bn, T, R, Cc = 3, 7, 20, 24
    al = torch.randn(Bn, T, R, device="cuda")
    dc = torch.randn(T, Bn, Cc, device="cuda")
    out = torch.randn(Bn, R, Cc, device="cuda")
    ref = out.double() + torch.einsum("btr,tbc->brc", al.double(), dc.double())
    _gemm(al, dc, out, R, Cc, T, 1, R, Bn * Cc, 1, Cc, batch=Bn, sA=T * R, sB=Cc, sC=R * Cc, acc=1)
    assert relerr(out, ref.float()) < 1e-5


def test_colsum():
    _lib, L = _L()
    X = torch.randn(1000, 70, device="cuda")
    o = torch.zeros(64, device="cuda")
    _lib.check(L.lo_colsum(_lib.ptr(X), 0, _lib.ptr(o), 1000, 64, 70, 0, _lib.stream_ptr()))
    assert relerr(o, X[:, :64].double().sum(0).float()) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum_vectorised_path(dtype):
    """N % 8 == 0, ld % 8 == 0, >= 256 rows: the 16-byte-per-lane kernel (bias gradients of the conv stack take this path)."""
    _lib, L = _L()
    torch.manual_seed(2)
    X = torch.randn(5000, 520, device="cuda").to(dtype)
    o = torch.full((512,), 7.0, device="cuda")
    _lib.check(L.lo_colsum(_lib.ptr(X), _lib.dt_of(X), _lib.ptr(o), 5000, 512, 520, 0, _lib.stream_ptr()))
    assert relerr(o, X[:, :512].double().sum(0).float()) < 1e-5
    _lib.check(L.lo_colsum(_lib.ptr(X), _lib.dt_of(X), _lib.ptr(o), 5000, 512, 520, 1, _lib.stream_ptr()))     # accumulate
    assert relerr(o, 2 * X[:, :512].double().sum(0).float()) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_conv1_pool(dtype):
    _lib, L = _L()
    torch.manual_seed(3)
    N, H, W = 2, 18, 38
    img = torch.randint(0, 256, (N, 1, H, W), device="cuda").float()
    w = torch.randn(64, 1, 3, 3, device="cuda") * 0.1
    b = torch.randn(64, device="cuda")
    out = torch.zeros(N, H // 2, W // 2, 64, device="cuda", dtype=dtype)
    _lib.check(L.lo_conv1_pool_forward(_lib.ptr(img), _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), _lib.dt_of(out), N, H, W, _lib.stream_ptr()))
    x = img.double()
    wr = w.double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    ref = F.max_pool2d(F.relu(F.conv2d(x, wr, br, padding=1)), 2)
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert relerr(out.float().permute(0, 3, 1, 2), ref) < tol
    if dtype == torch.float32:
        g = torch.randn_like(ref)
        ref.backward(g)
        dw = torch.zeros(64, 9, device="cuda")
        db = torch.zeros(64, device="cuda")
        gp = g.float().permute(0, 2, 3, 1).contiguous()
        _lib.check(L.lo_conv1_pool_wgrad(_lib.ptr(img), _lib.ptr(w), _lib.ptr(b), _lib.ptr(gp), 0, _lib.ptr(dw), _lib.ptr(db), N, H, W, _lib.stream_ptr()))
        assert relerr(dw.view(64, 1, 3, 3), wr.grad) < 1e-4
        assert relerr(db, br.grad) < 1e-4


@pytest.mark.parametrize("pad", [0, 1, 2])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_conv3x3_forward_dgrad_wgrad(pad, dtype):
    _lib, L = _L()
    torch.manual_seed(4 + pad)
    N, H, W, Cin, Cout = 2, 9, 13, 32, 80
    x = torch.randn(N, Cin, H, W, device="cuda")
    w = torch.randn(Cout, Cin, 3, 3, device="cuda") * 0.05
    b = torch.randn(Cout, device="cuda")
    xq, wq = x.to(dtype).float(), w.to(dtype).float()
    xr = xq.double().requires_grad_(True)
    wr = wq.double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    ref = F.relu(F.conv2d(xr, wr, br, padding=pad))          # float64: cuDNN fp32 would silently use TF32
    xn = xq.permute(0, 2, 3, 1).contiguous().to(dtype)
    wk = wq.permute(0, 2, 3, 1).contiguous().to(dtype)            # [Cout][3][3][Cin]
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    y = torch.zeros(N, Ho, Wo, Cout, device="cuda", dtype=dtype)
    st = _lib.stream_ptr()
    _lib.check(L.lo_conv3x3(_lib.ptr(xn), _lib.ptr(wk), _lib.ptr(b), None, _lib.ptr(y), _lib.dt_of(y), N, H, W, Cin, Cout, pad, 1, 0, st))
    tol = 1e-5 if dtype == torch.float32 else 1.5e-2
    assert relerr(y.float().permute(0, 3, 1, 2), ref) < tol
    # backward pieces against autograd
    g = torch.randn_like(ref).to(dtype).double()
    ref.backward(g)
    dy = (g * (ref > 0)).float().permute(0, 2, 3, 1).contiguous().to(dtype)          # dY (post ReLU mask)
    dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
    db = torch.zeros(Cout, device="cuda")
    _lib.check(L.lo_conv3x3_wgrad(_lib.ptr(xn), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db), _lib.dt_of(y), N, H, W, Cin, Cout, pad, 0, st))
    tolg = 1e-4 if dtype == torch.float32 else 2e-2
    assert relerr(dw.permute(0, 3, 1, 2), wr.grad) < tolg
    assert relerr(db, br.grad) < tolg
    wt = torch.zeros(Cin, 3, 3, Cout, device="cuda", dtype=dtype)
    _lib.check(L.lo_conv_weight_flip(_lib.ptr(wk), _lib.ptr(wt), _lib.dt_of(wk), Cin, Cout, st))
    dx = torch.zeros(N, H, W, Cin, device="cuda", dtype=dtype)
    _lib.check(L.lo_conv3x3(_lib.ptr(dy), _lib.ptr(wt), None, None, _lib.ptr(dx), _lib.dt_of(dx), N, Ho, Wo, Cout, Cin, 2 - pad, 0, 0, st))
    assert relerr(dx.float().permute(0, 3, 1, 2), xr.grad) < tolg


@pytest.mark.parametrize("k", [(2, 2), (2, 1), (1, 2)])
def test_maxpool(k):
    _lib, L = _L()
    torch.manual_seed(5)
    N, H, W, C = 2, 9, 10, 16
    x = torch.relu(torch.randn(N, C, H, W, device="cuda")).requires_grad_(True)
    ref = F.max_pool2d(x, k, k)
    g = torch.randn_like(ref)
    ref.backward(g)
    xn = x.detach().permute(0, 2, 3, 1).contiguous()
    y = torch.zeros(N, H // k[0], W // k[1], C, device="cuda")
    st = _lib.stream_ptr()
    _lib.check(L.lo_maxpool_forward(_lib.ptr(xn), _lib.ptr(y), 0, N, H, W, C, k[0], k[1], st))
    assert relerr(y.permute(0, 3, 1, 2), ref) == 0
    dy = g.permute(0, 2, 3, 1).contiguous()
    dx = torch.full((N, H, W, C), 7.0, device="cuda")
    _lib.check(L.lo_maxpool_backward(_lib.ptr(xn), _lib.ptr(y), _lib.ptr(dy), _lib.ptr(dx), 0, N, H, W, C, k[0], k[1], st))
    want = x.grad * (x.detach() > 0)            # fused ReLU mask
    assert relerr(dx.permute(0, 3, 1, 2), want) < 1e-6


@pytest.mark.parametrize("pipe", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,R", [(3, 37), (8, 180), (64, 868), (2, 5)])
def test_attention_forward(dtype, B, R, pipe):
    """pipe=1: TMA bulk-copy -> smem ring version (lo_attention.cu); pipe=0: register-streaming version."""
    _lib, L = _L()
    torch.manual_seed(6)
    C = A = 512
    enc = torch.randn(B, R, C, device="cuda").to(dtype)
    att1 = torch.randn(B, R, A, device="cuda").to(dtype)
    att2 = torch.randn(B, A + 16, device="cuda")[:, :A]          # strided rows
    wf = torch.randn(A, device="cuda") * 0.2
    gate_pre = torch.randn(B, C, device="cuda")
    gp0 = gate_pre.clone()
    alpha = torch.zeros(B, R, device="cuda")
    ctx = torch.zeros(B, C, device="cuda")
    gctx = torch.zeros(B, C, device="cuda")
    work = torch.zeros(int(L.lo_attention_workspace_bytes(B, C)), dtype=torch.uint8, device="cuda")
    with _lib.option(att_pipe=pipe):
        for _ in range(2):     # second launch checks that the ticket counters were reset
            gate_pre.copy_(gp0)
            _lib.check(L.lo_attention_forward(_lib.ptr(att1), _lib.ptr(enc), _lib.dt_of(enc), _lib.ptr(att2), att2.stride(0), _lib.ptr(wf),
                                              _lib.ptr(alpha), R, _lib.ptr(ctx), _lib.ptr(gate_pre), C, _lib.ptr(gctx), B, R, A, C,
                                              _lib.ptr(work), _lib.stream_ptr()))
            torch.cuda.synchronize()
    e = (torch.relu(att1.double() + att2.double()[:, None, :]) * wf.double()).sum(-1)
    al = torch.softmax(e, dim=1)
    cx = torch.einsum("br,brc->bc", al, enc.double())
    assert relerr(alpha, al.float()) < 2e-5
    assert relerr(ctx, cx.float()) < 2e-5
    assert relerr(gate_pre, torch.sigmoid(gp0)) < 1e-6
    assert relerr(gctx, (torch.sigmoid(gp0.double()) * cx).float()) < 2e-5


def test_adam_matches_torch():
    _lib, L = _L()
    torch.manual_seed(7)
    n = 10007
    p = torch.randn(n, device="cuda")
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-3)
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    state = torch.tensor([0.0, 1e-3], device="cuda")
    shadow = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        g = torch.randn(n, device="cuda")
        ref.grad = g.clone()
        opt.step()
        _lib.check(L.lo_adam_step(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), _lib.ptr(shadow), n, _lib.ptr(state),
                                  0.9, 0.999, 1e-8, 1.0, _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert (p - ref.detach()).abs().max().item() < 2e-6
    assert state[0].item() == 3.0
    assert relerr(shadow.float(), p) < 1e-2


def test_adam_ranges_skip_frozen_slices():
    """lo_adam_step_ranges == torch.optim.Adam over the un-frozen parameters only (frozen: no update, no moment decay)."""
    import ctypes
    _lib, L = _L()
    torch.manual_seed(8)
    sizes = (300, 1000, 77, 2048)
    frozen = (True, False, False, True)
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    n = offs[-1]
    p = torch.randn(n, device="cuda")
    p0 = p.clone()
    refs = [p[offs[i]:offs[i + 1]].clone().requires_grad_(True) for i in range(4)]
    opt = torch.optim.Adam([r for r, f in zip(refs, frozen) if not f], lr=2e-3)
    m = torch.randn(n, device="cuda").abs() * 1e-3          # stale moments on frozen slices must survive untouched
    v = torch.randn(n, device="cuda").abs() * 1e-3
    m[offs[1]:offs[3]] = 0
    v[offs[1]:offs[3]] = 0
    m0, v0 = m.clone(), v.clone()
    state = torch.tensor([0.0, 2e-3], device="cuda")
    ranges = (ctypes.c_int64 * 2)(offs[1], sizes[1] + sizes[2])
    for _ in range(3):
        g = torch.randn(n, device="cuda")
        for i in (1, 2):
            refs[i].grad = g[offs[i]:offs[i + 1]].clone()
        opt.step()
        _lib.check(L.lo_adam_step_ranges(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), None, ranges, 1, _lib.ptr(state),
                                         0.9, 0.999, 1e-8, 1.0, _lib.stream_ptr()))
    torch.cuda.synchronize()
    for i in range(4):
        sl = slice(offs[i], offs[i + 1])
        if frozen[i]:
            assert torch.equal(p[sl], p0[sl]) and torch.equal(m[sl], m0[sl]) and torch.equal(v[sl], v0[sl])
        else:
            assert (p[sl] - refs[i].detach()).abs().max().item() < 2e-6
    assert state[0].item() == 3.0


@pytest.mark.parametrize("kind", [1, 2, 3, 4])
def test_tf_optimisers_follow_tf_update_rules(kind):
    """lo_tf_optim_step: the four optimisers of model/img2seq.py:98-111 with TensorFlow 1.12's update rules restated in fp64
    (parity unpinned: TF cannot run here).  1 Adam (epsilon outside the bias correction), 2 SGD, 3 Adagrad (accumulator starts at
    0.1), 4 RMSProp (rms slot starts at 1, decay 0.9, epsilon 1e-10, momentum 0)."""
    _lib, L = _L()
    fn = L.lo_tf_optim_step
    torch.manual_seed(kind)
    n, lr = 5003, 1e-2
    p = torch.randn(n, device="cuda")
    ref = p.double().cpu()
    s1 = torch.full((n,), {1: 0.0, 2: 0.0, 3: 0.1, 4: 1.0}[kind], device="cuda")
    s2 = torch.zeros(n, device="cuda")
    r1, r2 = s1.double().cpu(), s2.double().cpu()
    state = torch.tensor([0.0, lr], device="cuda")
    b1, b2, eps = (0.9, 0.9, 1e-10) if kind == 4 else (0.9, 0.999, 1e-8)
    for t in range(1, 4):
        g = torch.randn(n, device="cuda")
        _lib.check(fn(kind, _lib.ptr(p), _lib.ptr(g), _lib.ptr(s1), _lib.ptr(s2), None, n, _lib.ptr(state), b1, b2, eps, 0.5, _lib.stream_ptr()))
        gd = g.double().cpu() * 0.5
        if kind == 1:
            r1 = b1 * r1 + (1 - b1) * gd
            r2 = b2 * r2 + (1 - b2) * gd * gd
            ref = ref - lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t) * r1 / (r2.sqrt() + eps)
        elif kind == 2:
            ref = ref - lr * gd
        elif kind == 3:
            r1 = r1 + gd * gd
            ref = ref - lr * gd / r1.sqrt()
        else:
            r1 = b2 * r1 + (1 - b2) * gd * gd
            ref = ref - lr * gd / (r1 + eps).sqrt()
    torch.cuda.synchronize()
    assert relerr(p, ref.float()) < 2e-6
    assert state[0].item() == 3.0
