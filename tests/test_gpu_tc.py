"""-m gpu: the wgmma/TMA kernels (lo_tc.cu) against float64 references and against the CUDA-core path."""
import pytest
import torch
import torch.nn.functional as F

from util import relerr

pytestmark = pytest.mark.gpu


def _L():
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    if not L.lo_tc_available():
        pytest.skip("wgmma path needs an sm_90 device")
    return _lib, L


@pytest.mark.parametrize("M,N,K,out_dtype", [(128, 128, 64, torch.float32), (300, 512, 512, torch.bfloat16),
                                              (55552 // 8, 512, 512, torch.bfloat16), (77, 200, 128, torch.float32), (64, 64, 256, torch.float32)])
def test_tc_gemm_nt(M, N, K, out_dtype):
    _lib, L = _L()
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    b = torch.randn(N, device="cuda")
    C = torch.full((M, N), 3.0, device="cuda", dtype=out_dtype)
    _lib.check(L.lo_gemm(_lib.ptr(A), 1, _lib.ptr(W), 1, _lib.ptr(C), _lib.dt_of(C), M, N, K, K, 1, 1, K, N, 1, 0, 0, 0, _lib.ptr(b), 0, 1, 1,
                         _lib.stream_ptr()))
    torch.cuda.synchronize()
    ref = torch.relu(A.double() @ W.double().t() + b.double())
    tol = 1e-5 if out_dtype == torch.float32 else 1e-2
    assert relerr(C.float(), ref.float()) < tol


@pytest.mark.parametrize("M,N,K,acc", [(64, 3072, 512, 0), (64, 2048, 512, 0), (64, 1024, 2048, 1), (64, 512, 1024, 1), (40, 1024, 576, 0),
                                         (1, 200, 64, 1), (17, 30, 2112, 0), (200, 500, 512, 0), (255, 500, 512, 1), (64, 256, 4608, 1)])
def test_skinny_mma_gemm(M, N, K, acc):
    """The decoder's per-step GEMM shapes (M = batch <= 64 rows, fp32 out) through the mma.sync kernel (lo_skinny.cu) and
    through the wgmma kernel (option skinny_mma=0): both against float64."""
    _lib, L = _L()
    torch.manual_seed(1)
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(N, K, device="cuda") * 0.1).bfloat16()
    b = torch.randn(N, device="cuda")
    base = torch.randn(M, N, device="cuda")
    ref = (A.double() @ W.double().t() + b.double() + (base.double() if acc else 0)).float()
    for opt in (1, 0):
        if opt == 0 and (K % 64 or N % 8):
            continue                                   # wgmma path constraints
        with _lib.option(skinny_mma=opt):
            C = base.clone()
            _lib.check(L.lo_gemm(_lib.ptr(A), 1, _lib.ptr(W), 1, _lib.ptr(C), _lib.dt_of(C), M, N, K, K, 1, 1, K, N, 1, 0, 0, 0, _lib.ptr(b), acc, 0,
                                 1, _lib.stream_ptr()))
            torch.cuda.synchronize()
        assert relerr(C, ref) < 1e-5, opt


def test_tc_train_step_matches_simt_bf16():
    from util import build_model, load_golden
    from oracle import ref_model as rm
    rec = load_golden("cfg1")
    c = rec["case"]
    pe, pd = rm.init_params(c["V"], seed=c["pseed"])
    img, formula = rm.synthetic_batch(c["B"], c["H"], c["W"], c["V"], c["tmin"], c["tmax"], seed=c["dseed"])
    B, T = c["B"], formula.shape[1] - 1
    out = {}
    for impl in ("simt", "tc"):
        m = build_model(c["V"], pe, pd, "bf16", impl=impl)
        loss = m._step_body(img.cuda(), formula.cuda(), [T] * B, None)
        torch.cuda.synchronize()
        out[impl] = (loss[0].item(), m.encoder.store.grad.clone(), m.decoder.store.grad.clone())
    assert abs(out["tc"][0] - rec["loss"]) / abs(rec["loss"]) < 3e-2
    assert abs(out["tc"][0] - out["simt"][0]) / abs(out["simt"][0]) < 5e-3
    for i in (1, 2):
        a, b = out["tc"][i], out["simt"][i]
        assert torch.isfinite(a).all()
        assert (a - b).norm().item() / (b.norm().item() + 1e-30) < 5e-2


@pytest.mark.parametrize("N,H,W,Cin,Cout,pad", [(2, 8, 128, 64, 128, 1), (3, 16, 64, 128, 256, 1), (2, 16, 64, 512, 512, 0),
                                                 (2, 6, 30, 256, 128, 1), (5, 9, 13, 64, 128, 1)])
def test_tc_conv3x3_wgrad(N, H, W, Cin, Cout, pad):
    _lib, L = _L()
    torch.manual_seed(2)
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    x = torch.randn(N, Cin, H, W, device="cuda").bfloat16()
    dy = torch.randn(N, Cout, Ho, Wo, device="cuda").bfloat16()
    w = torch.zeros(Cout, Cin, 3, 3, device="cuda", dtype=torch.float64, requires_grad=True)
    out = F.conv2d(x.double(), w, None, padding=pad)
    out.backward(dy.double())
    xn = x.permute(0, 2, 3, 1).contiguous()
    dyn = dy.permute(0, 2, 3, 1).contiguous()
    dw = torch.full((Cout, 3, 3, Cin), 9.0, device="cuda")
    db = torch.zeros(Cout, device="cuda")
    _lib.check(L.lo_conv3x3_wgrad(_lib.ptr(xn), _lib.ptr(dyn), _lib.ptr(dw), _lib.ptr(db), 1, N, H, W, Cin, Cout, pad, 1, _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert relerr(dw.permute(0, 3, 1, 2), w.grad.float()) < 2e-5        # bf16 inputs are exact in fp64; fp32 accumulate
    assert relerr(db, dy.double().sum(dim=(0, 2, 3)).float()) < 1e-5


_SCHEDULE_OPTS = {"skinny_mma": (1, 0), "att_maskbits": (1, 0), "wgrad256": (0, 1), "conv_mc": (1, 0), "att_bwd_mma": (1, 0),
                  "skinny_tma": (1, 0)}


@pytest.mark.parametrize("opt", sorted(_SCHEDULE_OPTS))
def test_optional_decoder_schedules_match_default(opt):
    """Every optional schedule (first value = default) must give the default schedule's numbers: the measured-no-faster variants kept
    as run-time options (DESIGN.md §8) and, the other way round, the paths the defaults replaced, such as the CUDA-core attention
    backward."""
    from util import build_model, load_golden
    from latex_ocr_b200 import _lib
    from oracle import ref_model as rm
    _L()
    V = 60
    pe, pd = rm.init_params(V, seed=41)
    img, formula = rm.synthetic_batch(40, 32, 64, V, 4, 6, seed=42)     # 40 rows: the per-step GEMMs (M <= 64) on mma.sync by default
    B, T = formula.shape[0], formula.shape[1] - 1
    res = {}
    for val in _SCHEDULE_OPTS[opt]:
        with _lib.option(**{opt: val}):
            m = build_model(V, pe, pd, "bf16", impl="tc")
            loss = m._step_body(img.cuda(), formula.cuda(), [T] * B, None)
            torch.cuda.synchronize()
            res[val] = (loss[0].item(), m.decoder.store.grad.clone())
    (l0, g0), (l1, g1) = res.values()
    assert abs(l0 - l1) / abs(l0) < 1e-4
    assert (g0 - g1).norm().item() / g0.norm().item() < 2e-2


def test_deterministic_option_gives_bit_identical_steps():
    """Option "deterministic": every cross-CTA reduction of the train step (split-K per-step GEMMs, weight gradients, bias column
    sums, the d w_full sweep, conv1's weight gradient) adds in a fixed order, so one full step (forward, backward, Adam) from the
    same parameters and inputs gives bitwise the same gradients and updated parameters.  The default mode's gradients (fp32
    atomics) must agree with it to rounding.  Also a per-step GEMM longer than one cluster of K slices (K > 8 x 512)."""
    from util import build_model, load_golden
    from oracle import ref_model as rm
    _lib, L = _L()
    rec = load_golden("cfg1")
    c = rec["case"]
    pe, pd = rm.init_params(c["V"], seed=c["pseed"])
    img, formula = rm.synthetic_batch(c["B"], c["H"], c["W"], c["V"], c["tmin"], c["tmax"], seed=c["dseed"])
    B, T = c["B"], formula.shape[1] - 1
    torch.manual_seed(3)
    A = torch.randn(64, 4608, device="cuda").bfloat16()
    W = (torch.randn(256, 4608, device="cuda") * 0.1).bfloat16()
    base = torch.randn(64, 256, device="cuda")
    ref = (A.double() @ W.double().t() + base.double()).float()
    runs = {}
    for det in (1, 1, 0):
        with _lib.option(deterministic=det):
            m = build_model(c["V"], pe, pd, "bf16", impl="tc")
            m._step_body(img.cuda(), formula.cuda(), [T] * B, None)
            C = base.clone()
            _lib.check(L.lo_gemm(_lib.ptr(A), 1, _lib.ptr(W), 1, _lib.ptr(C), 0, 64, 256, 4608, 4608, 1, 1, 4608, 256, 1, 0, 0, 0, None, 1,
                                 0, 1, _lib.stream_ptr()))
            torch.cuda.synchronize()
        assert relerr(C, ref) < 1e-5, det
        stores = (m.encoder.store, m.decoder.store)
        runs.setdefault(det, []).append([t.clone() for s_ in stores for t in (s_.grad, s_.master)] + [C])
    first, second = runs[1]
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    # against the default mode, parameter by parameter: the gradients differ by the rounding of the summation order, which the
    # bf16 storage of the backward activations can raise to one bf16 ulp (2^-8) on single elements (measured: <= 1e-3 norm-wise,
    # the same as between two runs of the default mode)
    assert relerr(first[4], runs[0][0][4]) < 1e-6
    for i, s_ in ((0, m.encoder.store), (2, m.decoder.store)):
        for name, (off, n, _) in s_.offsets.items():
            a, b = first[i][off:off + n], runs[0][0][i][off:off + n]
            assert (a - b).norm().item() <= 5e-3 * b.norm().item() + 1e-9, name
