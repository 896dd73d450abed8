"""CPU: the per-step float64 restatement of the sequence LSTM (tests/lstmseq_step_ref.py), chained over S steps, reproduces
oracle/ref_ext.lstm_seq and torch.nn.LSTM (with an initial state) and their float64 autograd gradients.
tests/test_gpu_lstmseq_steps.py compares the kernels with the pieces of that restatement one launch at a time; this test is what
ties those pieces to the definition.  Also: the restated workspace layout is the library's, and lo_lstm_seq_forward / _backward
refuse x and dx that their 16-byte loads and stores could not serve."""
import ctypes

import pytest
import torch

import lstmseq_step_ref as lr
from oracle import ref_ext as rx


def _params(seed, M, S, I, H):
    g = torch.Generator().manual_seed(seed)
    b = 1.0 / H ** 0.5

    def U(*shape):
        return (torch.rand(*shape, generator=g, dtype=torch.float64) * 2 - 1) * b
    w_ih, w_hh, b_ih, b_hh = U(4 * H, I), U(4 * H, H), U(4 * H), U(4 * H)
    x = torch.randn(M, S, I, generator=g, dtype=torch.float64)
    dhs = torch.randn(M, S, H, generator=g, dtype=torch.float64)
    return w_ih, w_hh, b_ih, b_hh, x, dhs, g


def _close(a, b, what):
    err = (a - b).abs().max().item()
    assert err <= 1e-12 * max(1.0, b.abs().max().item()), (what, err)


@pytest.mark.parametrize("reverse", [False, True], ids=["forward", "reverse"])
def test_chained_steps_match_the_oracle(reverse):
    M, S, I, H = 3, 6, 10, 7
    w_ih, w_hh, b_ih, b_hh, x, dhs, g = _params(5 + reverse, M, S, I, H)
    base = torch.randn(M, S, I, generator=g, dtype=torch.float64)
    ps = [t.clone().requires_grad_(True) for t in (x, w_ih, w_hh, b_ih, b_hh)]
    out = rx.lstm_seq(ps[0], *ps[1:], reverse=reverse)
    (out * dhs).sum().backward()
    hs, _, gr = lr.chained(x, w_ih, w_hh, b_ih, b_hh, reverse, dhs=dhs, dx_base=base)
    _close(hs, out.detach(), "hs")
    _close(gr["dx"] - base, ps[0].grad, "dx")
    for k, p in (("g_w_ih", ps[1]), ("g_w_hh", ps[2]), ("g_b", ps[3]), ("g_b", ps[4])):
        _close(gr[k], p.grad, k)
    # without d hs every gradient is zero
    _, _, g0 = lr.chained(x, w_ih, w_hh, b_ih, b_hh, reverse)
    for k, v in g0.items():
        assert bool((v == 0).all()), k


@pytest.mark.parametrize("reverse", [False, True], ids=["forward", "reverse"])
def test_chained_steps_match_nn_lstm_with_an_initial_state(reverse):
    M, S, I, H = 4, 5, 8, 6
    w_ih, w_hh, b_ih, b_hh, x, dhs, g = _params(11 + reverse, M, S, I, H)
    h0 = 0.5 * torch.randn(M, H, generator=g, dtype=torch.float64)
    c0 = torch.randn(M, H, generator=g, dtype=torch.float64)
    lstm = torch.nn.LSTM(I, H, batch_first=True).double()
    with torch.no_grad():
        for n, v in (("weight_ih_l0", w_ih), ("weight_hh_l0", w_hh), ("bias_ih_l0", b_ih), ("bias_hh_l0", b_hh)):
            getattr(lstm, n).copy_(v)
    xr, h0r, c0r = (t.clone().requires_grad_(True) for t in (x, h0, c0))
    flip = (lambda t: t.flip(1)) if reverse else (lambda t: t)       # the reverse direction is nn.LSTM over the flipped sequence
    out, _ = lstm(flip(xr), (h0r[None], c0r[None]))
    (flip(out) * dhs).sum().backward()
    hs, _, gr = lr.chained(x, w_ih, w_hh, b_ih, b_hh, reverse, h0=h0, c0=c0, dhs=dhs)
    _close(hs, flip(out).detach(), "hs")
    _close(gr["dx"], xr.grad, "dx")
    _close(gr["dh0"], h0r.grad, "dh0")
    _close(gr["dc0"], c0r.grad, "dc0")
    _close(gr["g_w_ih"], lstm.weight_ih_l0.grad, "g_w_ih")
    _close(gr["g_w_hh"], lstm.weight_hh_l0.grad, "g_w_hh")
    _close(gr["g_b"], lstm.bias_ih_l0.grad, "g_b_ih")
    _close(gr["g_b"], lstm.bias_hh_l0.grad, "g_b_hh")


# ---- the workspace layout
_SHAPES = [  # (S, M, I, H)
    (78, 36, 512, 256),      # the row encoder at N = 2
    (7, 72, 512, 512),       # layer 2
    (5, 520, 48, 80),
    (4, 65, 64, 128),
    (1, 1, 8, 8),
    (9, 3, 24, 40),
]


def _args(S, M, I, H, bf16):
    from latex_ocr_b200 import _lib
    a = _lib.LstmSeqArgs()
    a.S, a.M, a.I, a.H = S, M, I, H
    a.dt = _lib.dtype_code("bf16" if bf16 else "fp32")
    return a


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_workspace_layout_is_the_librarys(bf16):
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    for S, M, I, H in _SHAPES:
        _, end = lr.carve(S, M, I, H, bf16)
        assert int(L.lo_lstm_seq_workspace_bytes(ctypes.byref(_args(S, M, I, H, bf16)))) == end, (S, M, I, H)


# ---- refusals before any GPU work (the pointers are never dereferenced)
def _valid(backward):
    a = _args(3, 2, 16, 8, True)
    a.x, a.w_ih, a.w_hh, a.b_ih, a.b_hh, a.ws = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000, 0x6000
    a.x_row, a.x_step = 48, 16
    a.hs_st, a.hs_row, a.hs_step = 0x7000, 24, 8
    if backward:
        a.g_w_ih, a.g_w_hh, a.g_b_ih, a.g_b_hh = 0x8000, 0x9000, 0xa000, 0xb000
        a.dx, a.dx_row, a.dx_step = 0xc000, 48, 16
    return a


def _call(a, backward):
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    rc = L.lo_lstm_seq_backward(ctypes.byref(a), None) if backward else L.lo_lstm_seq_forward(ctypes.byref(a), None)
    return rc, L.lo_last_error()


@pytest.mark.parametrize("backward", [False, True], ids=["forward", "backward"])
def test_misaligned_x_is_refused(backward):
    for off in (2, 8):
        a = _valid(backward)
        a.x += off
        rc, err = _call(a, backward)
        assert rc == -1 and b"x must be 16-byte aligned" in err, (off, rc, err)


@pytest.mark.parametrize("field,value,message", [
    ("dx", 0xc008, b"dx must be 16-byte aligned"),
    ("dx", 0xc004, b"dx must be 16-byte aligned"),
    ("dx_row", 46, b"dx strides must be multiples of 4"),
    ("dx_step", 18, b"dx strides must be multiples of 4"),
])
def test_misaligned_dx_is_refused(field, value, message):
    a = _valid(True)
    setattr(a, field, value)
    rc, err = _call(a, True)
    assert rc == -1 and message in err, (field, rc, err)
    # without dx the backward writes no d x, so its strides are not looked at
    a = _valid(True)
    a.dx, a.dx_row, a.dx_step = None, 3, 5
    a.g_w_ih = None
    rc, err = _call(a, True)
    assert rc == -1 and b"null gradient buffer" in err, err
