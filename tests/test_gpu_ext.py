"""-m gpu: the EXTENSION (BASELINE.json configs[3]: row-encoder biLSTM + second decoder layer, latex_ocr_b200/ext.py) against its CPU
definition oracle/ref_ext.py (torch's own LSTM arithmetic + the pinned restatement of encoder / attention / loss; "parity
unpinned — extension": the reference has no such model).  fp32: loss 1e-4, gradients 1e-3 of max-abs; bf16: stated loose bounds."""
import pytest
import torch

from util import Cfg, relerr

pytestmark = pytest.mark.gpu


def _seq_case(dtype, S, M, I, H, reverse, seed):
    """One direction through the C ABI on a [M][S][I] batch-major tensor vs oracle/ref_ext.lstm_seq + autograd."""
    import ctypes
    from latex_ocr_b200 import _lib, ext
    from latex_ocr_b200.params import FlatStore
    from oracle import ref_ext as rx
    g = torch.Generator().manual_seed(seed)
    b = 1.0 / H ** 0.5
    p = {"weight_ih": (torch.rand(4 * H, I, generator=g) * 2 - 1) * b, "weight_hh": (torch.rand(4 * H, H, generator=g) * 2 - 1) * b,
         "bias_ih": (torch.rand(4 * H, generator=g) * 2 - 1) * b, "bias_hh": (torch.rand(4 * H, generator=g) * 2 - 1) * b}
    x = torch.randn(M, S, I, generator=g)
    dh = torch.randn(M, S, H, generator=g)
    precision = "fp32" if dtype == torch.float32 else "bf16"
    store = FlatStore([("l.weight_ih", (4 * H, I)), ("l.weight_hh", (4 * H, H)), ("l.bias_ih", (4 * H,)), ("l.bias_hh", (4 * H,))], "cuda",
                      bf16_shadow=(precision == "bf16"))
    for k, v in p.items():
        store.f32("l." + k).copy_(v)
    store.sync_shadow()
    if precision == "bf16":                      # the oracle sees what the kernels see: bf16-rounded weights and inputs
        p = {k: (v.bfloat16().float() if k.startswith("weight") else v) for k, v in p.items()}
        x = x.bfloat16().float()
    d = ext._Direction(store, "l.", "", I, H, precision, "tc" if precision == "bf16" else "simt", reverse)
    a = d.args(S, M)
    xd = x.cuda().to(dtype).contiguous()
    hs = torch.zeros(M, S, H, device="cuda")
    dx = torch.zeros(M, S, I, device="cuda")
    dhd = dh.cuda().contiguous()
    a.x, a.x_row, a.x_step = xd.data_ptr(), S * I, I
    a.hs, a.hs_st, a.hs_row, a.hs_step = hs.data_ptr(), None, S * H, H
    L = ext._bind()
    _lib.check(L.lo_lstm_seq_forward(ctypes.byref(a), _lib.stream_ptr()))
    a.dhs, a.dx, a.dx_row, a.dx_step, a.dx_accumulate = dhd.data_ptr(), dx.data_ptr(), S * I, I, 0
    _lib.check(L.lo_lstm_seq_backward(ctypes.byref(a), _lib.stream_ptr()))
    torch.cuda.synchronize()
    pr = {k: v.double().requires_grad_(True) for k, v in p.items()}
    xr = x.double().requires_grad_(True)
    out = rx.lstm_seq(xr, pr["weight_ih"], pr["weight_hh"], pr["bias_ih"], pr["bias_hh"], reverse=reverse)
    (out * dh.double()).sum().backward()
    return hs, out, dx, xr.grad, {k: store.g("l." + k).clone() for k in p}, {k: v.grad for k, v in pr.items()}


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("S,M,I,H", [(5, 7, 64, 64), (9, 70, 128, 64)])
def test_lstm_seq_fp32_matches_torch(S, M, I, H, reverse):
    hs, out, dx, dxr, g, gr = _seq_case(torch.float32, S, M, I, H, reverse, seed=S + M)
    assert relerr(hs, out) < 1e-5
    assert relerr(dx, dxr) < 1e-4
    for k in g:
        assert relerr(g[k], gr[k]) < 1e-4, k


@pytest.mark.parametrize("S,M,I,H", [(6, 48, 128, 64), (7, 200, 512, 256)])
def test_lstm_seq_bf16_tensor_core_path(S, M, I, H):
    """bf16 storage + wgmma / mma.sync GEMMs (M <= 64 and M > 64 both), inputs pre-rounded so only the kernels' own
    rounding (bf16 mirrors of h and d pre-activations) shows: STATED tolerance 2e-2 of max-abs."""
    hs, out, dx, dxr, g, gr = _seq_case(torch.bfloat16, S, M, I, H, False, seed=S * 3 + M)
    assert relerr(hs, out) < 2e-2
    assert relerr(dx, dxr) < 2e-2
    for k in g:
        assert relerr(g[k], gr[k]) < 2e-2, k


def _ext_model(V, pe, prow, pd, p2, precision, train=False):
    from latex_ocr_b200.ext import Img2SeqRowModel
    m = Img2SeqRowModel(Cfg(), n_tok=V, device="cuda", precision=precision, impl="tc" if precision == "bf16" else "simt")
    m.build_train()
    m.encoder.load_state_dict(pe)
    m.decoder.load_state_dict(pd)
    m.row_encoder.load_state_dict(prow)
    m.layer2.load_state_dict(p2)
    m.train_mode(train)
    return m


def test_row_encoder_module_matches_nn_lstm():
    from latex_ocr_b200.ext import RowEncoder
    from oracle import ref_ext as rx
    prow, _ = rx.init_params_ext(seed=2)
    enc = RowEncoder(512, 256, precision="fp32")
    assert set(enc.state_dict()) == set(prow)
    enc.load_state_dict(prow)
    feat = torch.randn(2, 3, 9, 512, generator=torch.Generator().manual_seed(3))
    lstm = torch.nn.LSTM(512, 256, bidirectional=True, batch_first=True)
    lstm.load_state_dict({k.split(".", 1)[1]: v for k, v in prow.items()})
    want, _ = lstm(feat.reshape(6, 9, 512))
    got = enc(feat.cuda())
    assert got.shape == (2, 3, 9, 512) and relerr(got.reshape(6, 9, 512), want) < 1e-5


def test_ext_train_step_fp32_vs_oracle_all_gradients():
    """Whole extension model (CNN -> row biLSTM -> 2-layer attention decoder -> loss -> backward), dropout multipliers injected."""
    from oracle import ref_ext as rx
    from oracle import ref_model as rm
    V = 50
    pe, pd = rm.init_params(V, seed=7)
    prow, p2 = rx.init_params_ext(seed=8)
    img, formula = rm.synthetic_batch(3, 40, 72, V, 4, 7, seed=9)
    B, T = formula.shape[0], formula.shape[1] - 1
    mask = (torch.rand(B, T, 512, generator=torch.Generator().manual_seed(5)) >= 0.5).float() * 2.0
    want, (ge, grow, gd, g2), aux = rx.train_grads_ext(pe, prow, pd, p2, img, formula, mask)
    m = _ext_model(V, pe, prow, pd, p2, "fp32", train=True)
    loss = m._step_body(img.cuda(), formula.cuda(), [T] * B, mask.cuda())
    torch.cuda.synchronize()
    assert abs(loss[0].item() - want) / abs(want) < 1e-4, (loss[0].item(), want)
    for mod, ref in ((m.decoder, gd), (m.layer2, g2), (m.row_encoder, grow), (m.encoder, ge)):
        for k, p_ in mod.named_parameters():
            if k == "attention.full_att.bias":
                continue
            g = p_.grad.detach().float().cpu()
            err = (g.double() - ref[k].double()).abs().max().item()
            assert err <= 1e-3 * ref[k].abs().max().item() + 2e-8, (k, err, ref[k].abs().max().item())


def test_ext_bf16_close_to_oracle_and_trains():
    """bf16 / wgmma path of the extension: STATED tolerance loss 5e-3 relative; repeated steps on one batch reduce the loss;
    the CUDA-graph step equals the eager one."""
    from oracle import ref_ext as rx
    from oracle import ref_model as rm
    V = 50
    pe, pd = rm.init_params(V, seed=7)
    prow, p2 = rx.init_params_ext(seed=8)
    img, formula = rm.synthetic_batch(4, 32, 64, V, 4, 6, seed=10)
    B, T = formula.shape[0], formula.shape[1] - 1
    want, _ = rx.get_loss_ext(pe, prow, pd, p2, img, formula)
    m = _ext_model(V, pe, prow, pd, p2, "bf16")
    loss = m._step_body(img.cuda(), formula.cuda(), [T] * B, None)
    torch.cuda.synchronize()
    assert abs(loss[0].item() - want.item()) / abs(want.item()) < 5e-3, (loss[0].item(), want.item())
    m.train_mode(True)
    first = -m.getLoss(img, formula)
    for _ in range(12):
        last = -m.getLoss(img, formula)
    assert last < first, (first, last)
    with pytest.raises(NotImplementedError):
        m.predict_batch(img)
