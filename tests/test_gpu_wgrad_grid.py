"""-m gpu: the weight-gradient kernel's split-K decompositions (lo_tc.cu, tc_wgrad_kernel) against float64 on the kernel's own
bf16 inputs.  Default mode: whole-wave grids, one split or several, the last one ragged.  Option "deterministic": the ordered
cluster sum of up to 8 splits, bit-identical from call to call.  Convolutions with Cin of 256 and 512 run the 128 x 256 tiles on
64-position K blocks, and so does the TN GEMM with N % 256 == 0 under option wgrad256; the others run 128 x 128 / 128 x 64
tiles on 128-position blocks.  The convolution cases also run the CUDA-core kernel (fp32 storage, and bf16 with
conv_impl="simt"), whose position splits must be just as reproducible under "deterministic"."""
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


# (N, H, W, Cin, Cout, pad): one split (2 K blocks); 8 splits in both modes; 128-channel tiles with an 8-split cluster; 128 x 256
# tiles cutting 64 x 2 boxes into row halves (pad 0); 16 x 8 boxes with out-of-bounds rows and columns; Cin 512 at pad 0; rows
# of 140 positions (two 128-wide boxes cut into column halves) with a ragged last split
CONVS = [(1, 6, 30, 64, 128, 1), (4, 16, 64, 64, 128, 1), (2, 16, 64, 128, 256, 1), (2, 12, 40, 256, 256, 0), (3, 9, 13, 256, 128, 1),
         (2, 10, 34, 512, 256, 0), (2, 4, 140, 512, 128, 1)]


# impl: the tensor-core kernel (bf16), or the CUDA-core kernel (conv3x3_wgrad_kernel) at fp32 and at bf16.  The CUDA-core kernel
# cuts the positions into up to cdiv(528, 9 cdiv(Cin, 64) cdiv(Cout, 64)) splits of at least 512 positions each, added with
# atomics; under "deterministic" at most two, whose two addends onto the zeroed dw sum the same in either order.
IMPLS = [("tc", "bf16"), ("simt", "fp32"), ("simt", "bf16")]


@pytest.mark.parametrize("impl,precision", IMPLS, ids=["%s_%s" % i for i in IMPLS])
@pytest.mark.parametrize("N,H,W,Cin,Cout,pad", CONVS)
def test_conv3x3_wgrad_splits_against_float64(N, H, W, Cin, Cout, pad, impl, precision):
    _lib, L = _L()
    g = torch.Generator(device="cuda").manual_seed(5)
    Ho, Wo = H + 2 * pad - 2, W + 2 * pad - 2
    dtype = torch.bfloat16 if precision == "bf16" else torch.float32
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).bfloat16().to(dtype)
    dy = torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g).bfloat16().to(dtype)
    w = torch.zeros(Cout, Cin, 3, 3, device="cuda", dtype=torch.float64, requires_grad=True)
    F.conv2d(x.permute(0, 3, 1, 2).double(), w, None, padding=pad).backward(dy.permute(0, 3, 1, 2).double())
    ref = w.grad.permute(0, 2, 3, 1)

    def run():
        dw = torch.full((Cout, 3, 3, Cin), 7.0, device="cuda")      # the call clears it
        _lib.check(L.lo_conv3x3_wgrad(_lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), None, _lib.dt_of(x), N, H, W, Cin, Cout, pad,
                                      _lib.impl_code(impl, precision), _lib.stream_ptr()))
        torch.cuda.synchronize()
        return dw

    assert relerr(run(), ref) < 1e-5
    with _lib.option(deterministic=1):
        a, b = run(), run()
    assert relerr(a, ref) < 1e-5
    assert torch.equal(a, b)


# (M, N, K): K tails of 1000 - 15 * 64 and 3000 - 46 * 64 positions; one K block of 70 positions (N = 64); ragged last splits at
# the decoder's one-hot^T dG and datt1^T enc shapes with smaller K
GEMMS = [(256, 512, 1000), (200, 200, 3000), (128, 64, 70), (504, 2048, 2400), (512, 512, 16 * 868)]


@pytest.mark.parametrize("wgrad256", [0, 1])
@pytest.mark.parametrize("M,N,K", GEMMS)
def test_gemm_tn_splits_against_float64(M, N, K, wgrad256):
    """C[M][N] = A[K][M]^T B[K][N] through lo_gemm's tensor-core route to the TN weight-gradient kernel (operands stored [K][.])."""
    _lib, L = _L()
    g = torch.Generator(device="cuda").manual_seed(6)
    A = torch.randn(K, M, device="cuda", generator=g).bfloat16()
    B = torch.randn(K, N, device="cuda", generator=g).bfloat16()
    ref = A.double().t() @ B.double()

    def run():
        C = torch.full((M, N), 7.0, device="cuda")
        _lib.check(L.lo_gemm(_lib.ptr(A), _lib.LO_BF16, _lib.ptr(B), _lib.LO_BF16, _lib.ptr(C), _lib.LO_F32, M, N, K, 1, M, N, 1, N,
                             1, 0, 0, 0, None, 0, 0, _lib.LO_IMPL_TC, _lib.stream_ptr()))
        torch.cuda.synchronize()
        return C

    with _lib.option(wgrad256=wgrad256):
        assert relerr(run(), ref) < 1e-5
        with _lib.option(deterministic=1):
            a, b = run(), run()
    assert relerr(a, ref) < 1e-5
    assert torch.equal(a, b)
