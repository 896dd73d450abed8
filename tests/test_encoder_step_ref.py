"""CPU: the per-launch float64 restatement of the encoder (tests/encoder_step_ref.py), chained in EncoderCNN's launch order,
reproduces oracle/ref_model.encoder_forward and its float64 autograd parameter gradients.  tests/test_gpu_encoder_steps.py
compares the kernels with the pieces of that restatement one launch at a time; this test is what ties those pieces to the
reference."""
import pytest
import torch

import encoder_step_ref as es
from oracle import ref_model as rm


def _layers(variant):
    # EncoderCNN's layer tables, restated here so that this test needs no part of the package beyond the oracle:
    # (sequential index, Cin, Cout, pad, pool after[, (R, S, stride)])
    if variant == "vanilla":
        return (("0", 1, 64, 1, (2, 2)), ("3", 64, 128, 1, (2, 2)), ("6", 128, 256, 1, None),
                ("8", 256, 256, 1, (2, 1)), ("11", 256, 512, 1, (1, 2)), ("14", 512, 512, 0, None))
    return (("0", 1, 64, 1, (2, 2)), ("3", 64, 128, 1, (2, 2)), ("6", 128, 256, 1, None), ("8", 256, 256, 1, None),
            ("10", 256, 512, 1, None), ("12", 512, 512, 1, None, (2, 4, 2)), ("14", 512, 512, 0, None))


def formula_images(N, H, W, g):
    """Formula-like integer pixels: 255 background, dark horizontal and vertical strokes on a few percent of the pixels; the
    last image is all white.  Flat white regions make the four conv positions of a pool window tie exactly."""
    img = torch.full((N, 1, H, W), 255.0)
    for n in range(N - 1):
        for _ in range(max(1, H * W // 400)):
            y, x = int(torch.randint(0, H, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g))
            ln = int(torch.randint(2, 12, (1,), generator=g))
            v = float(torch.randint(0, 120, (1,), generator=g))
            if torch.rand(1, generator=g).item() < 0.5:
                img[n, 0, y, x:x + ln] = v
            else:
                img[n, 0, y:y + ln, x] = v
    return img


@pytest.mark.parametrize("norm", [None, "tf"], ids=["raw", "tf"])
@pytest.mark.parametrize("positional", [True, False], ids=["pos", "nopos"])
@pytest.mark.parametrize("variant", ["vanilla", "cnn"])
def test_chained_launches_match_the_reference(variant, positional, norm):
    g = torch.Generator().manual_seed(len(variant) * 4 + 2 * positional + (norm is not None))
    N, H, W = (2, 27, 45) if variant == "vanilla" else (2, 32, 66)
    pe, _ = rm.init_params(10, seed=3, dtype=torch.float64, encoder_cnn=variant)
    for k in pe:                    # biases away from their small init, so that both sides of every ReLU are exercised
        if k.endswith("bias"):
            pe[k] = pe[k] + 0.05 * torch.randn(pe[k].shape, generator=g, dtype=torch.float64)
    img = formula_images(N, H, W, g)
    # a patch without ties, on a 1/256 grid so that the kernels' fp32 normalisation fmaf(img, 1/128, -1) is exact
    img[0, 0, :H // 2, :W // 3] = (torch.rand(H // 2, W // 3, generator=g) * 255 * 256).round() / 256

    p = {k: v.clone().requires_grad_(True) for k, v in pe.items()}
    xin = img.double() if norm is None else (img.double() - 128.0) / 128.0
    out = rm.encoder_forward(p, xin, positional, encoder_cnn=variant)
    denc = torch.randn(out.shape, generator=g, dtype=torch.float64)
    (out * denc).sum().backward()

    kp = {k: (v.permute(0, 2, 3, 1).contiguous() if v.dim() == 4 else v) for k, v in pe.items()}
    table = rm.timing_signal_nd(512, out.shape[1], out.shape[2], torch.float64).permute(1, 2, 0) if positional else None
    scale, offset = (1.0 / 128.0, -1.0) if norm == "tf" else (1.0, 0.0)
    out2, acts, grads, pg = es.chain(_layers(variant), kp, img, denc, table, scale, offset)

    def close(a, b, what):
        err = (a - b).abs().max().item()
        assert err <= 1e-12 * max(1.0, b.abs().max().item()), (what, err)

    close(out2, out.detach(), "encoder output")
    for k, v in p.items():
        close(pg[k], v.grad.permute(0, 2, 3, 1) if v.dim() == 4 else v.grad, k)
    assert all(v.grad.abs().max() > 0 for v in p.values())
    # the ties the kernels' first-maximum rule decides are there: whole windows of equal conv1 values
    _, _, v, _ = es.conv1_pool(es.pixels(img, scale, offset), kp["cnn.0.weight"], kp["cnn.0.bias"])
    assert ((v == v[..., :1]).all(-1) & (v[..., 0] > 0)).any()


def test_pieces_against_torch():
    """Spot checks of single pieces against torch's own operators where one exists: the code-routed conv1 weight gradient
    against autograd through conv2d + ReLU + max_pool2d, the max-pool backward, im2col / col2im and the strided conv's GEMMs."""
    g = torch.Generator().manual_seed(7)
    N, H, W = 2, 9, 13
    x = torch.randn(N, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(64, 1, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(64, generator=g, dtype=torch.float64, requires_grad=True)
    P0, arg, v, _ = es.conv1_pool(x, w.detach(), b.detach())
    code = (arg | torch.where(v.max(-1).values > 0, 4, 0)).to(torch.uint8)
    y = torch.nn.functional.max_pool2d(torch.relu(torch.nn.functional.conv2d(x[:, None], w, b, padding=1)), 2)
    assert torch.allclose(y.permute(0, 2, 3, 1), P0, rtol=0, atol=1e-13)
    dp = torch.randn(P0.shape, generator=g, dtype=torch.float64)
    (y * dp.permute(0, 3, 1, 2)).sum().backward()
    dw, _, db, _ = es.conv1_wgrad(x, code, dp)
    assert torch.allclose(dw, w.grad.reshape(64, 9), rtol=0, atol=1e-12) and torch.allclose(db, b.grad, rtol=0, atol=1e-12)

    for kh, kw in ((2, 2), (2, 1), (1, 2)):
        ya = torch.relu(torch.randn(N, H, W, 16, generator=g, dtype=torch.float64)).requires_grad_(True)
        pa = torch.nn.functional.max_pool2d(ya.permute(0, 3, 1, 2), (kh, kw))
        dpa = torch.randn(pa.shape, generator=g, dtype=torch.float64)
        (pa * dpa).sum().backward()
        assert torch.equal(es.maxpool(ya.detach(), kh, kw), pa.detach().permute(0, 2, 3, 1))
        # relu'(0) = 0: where the window's maximum is 0 the kernels write 0; torch routes to a zero of the ReLU output
        got = es.maxpool_backward(ya.detach(), dpa.permute(0, 2, 3, 1), kh, kw)
        assert torch.equal(got, ya.grad * (ya.detach() > 0))

    xc = torch.randn(N, 8, 10, 16, generator=g, dtype=torch.float64)
    wc = torch.randn(24, 2, 4, 16, generator=g, dtype=torch.float64)
    bc = torch.randn(24, generator=g, dtype=torch.float64)
    col = es.im2col(xc, 2, 4, 2, 1)
    yc = es.gemm_nt(col, wc.reshape(24, -1), bc)[0]
    ref = torch.nn.functional.conv2d(xc.permute(0, 3, 1, 2), wc.permute(0, 3, 1, 2), bc, stride=2, padding=1)
    assert torch.allclose(yc.view(N, ref.shape[2], ref.shape[3], 24), ref.permute(0, 2, 3, 1), rtol=0, atol=1e-12)
    xt = xc.clone().requires_grad_(True)
    wt = wc.permute(0, 3, 1, 2).clone().requires_grad_(True)
    yt = torch.nn.functional.conv2d(xt.permute(0, 3, 1, 2), wt, None, stride=2, padding=1)
    dy = torch.randn(yt.shape, generator=g, dtype=torch.float64)
    (yt * dy).sum().backward()
    dy2 = dy.permute(0, 2, 3, 1).reshape(-1, 24)
    assert torch.allclose(es.gemm_tn(dy2, col)[0].view(24, 2, 4, 16), wt.grad.permute(0, 2, 3, 1), rtol=0, atol=1e-12)
    assert torch.allclose(es.colsum(dy2)[0], dy.sum((0, 2, 3)), rtol=0, atol=1e-12)
    dcol = es.gemm_nn(dy2, wc.reshape(24, -1))[0]
    assert torch.allclose(es.col2im(dcol, None, N, 8, 10, 16, 2, 4, 2, 1)[0], xt.grad, rtol=0, atol=1e-12)
