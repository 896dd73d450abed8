"""CPU: the per-step float64 restatement of the TensorFlow-flavour decoder (tests/tfdec_step_ref.py), chained over T steps,
reproduces oracle/ref_tf_model.py's teacher-forced pass and masked cross entropy and their float64 autograd gradients.
tests/test_gpu_tfdec_steps.py compares the kernels with the pieces of that restatement one step at a time; this test is what ties
those pieces to the reference.  Also: the restated workspace layout (tfdec_step_ref.carve) is the library's."""
import ctypes

import pytest
import torch

import tfdec_step_ref as tr
from oracle import ref_tf_model as rt

_DIMS = dict(num_units=12, dim_e=10, dim_o=9, dim_embeddings=8, channels=14)


def _case(seed, keep, sampling):
    B, R, T, V = 3, 7, 5, 13
    p = rt.init_params_tf(V, seed=seed, dims=_DIMS, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed + 1)
    p["lstm.bias"] = 0.3 * torch.randn(p["lstm.bias"].shape, generator=g, dtype=torch.float64)     # away from its zero init
    enc = torch.randn(B, R, _DIMS["channels"], generator=g, dtype=torch.float64)
    formula = torch.randint(0, V, (B, T), generator=g)
    lengths = torch.tensor([T, 3, 1])
    keep_h = keep_o = fed = None
    if keep:
        keep_h = (torch.rand(B, T, _DIMS["num_units"], generator=g) >= 0.4).double() / 0.6
        keep_o = (torch.rand(B, T, _DIMS["dim_o"], generator=g) >= 0.4).double() / 0.6
    if sampling:
        fed = torch.randint(0, V, (B, T), generator=g)
    return p, enc, formula, lengths, keep_h, keep_o, fed


@pytest.mark.parametrize("keep,sampling", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["plain", "keep-masks", "sampling", "keep-masks-sampling"])
def test_chained_steps_match_the_reference(keep, sampling):
    p, enc, formula, lengths, keep_h, keep_o, fed = _case(3 + 2 * keep + sampling, keep, sampling)
    T = formula.shape[1]
    V = p["y_W_o"].shape[1]
    # the reference: the tokens consumed are those of its formula argument shifted behind the start token, the targets formula
    pr = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    x = enc.clone().requires_grad_(True)
    lg_ref, al_ref = rt.decoder_train_logits(pr, x, formula if fed is None else fed, keep_h, keep_o)
    loss_ref, _, _ = rt.masked_ce(lg_ref, formula, lengths)
    loss_ref.backward()
    loss, st, g = tr.chained(p, enc, formula, lengths, keep_h, keep_o, fed)

    def close(a, b, what):
        err = (a - b).abs().max().item()
        assert err <= 1e-12 * max(1.0, b.abs().max().item()), (what, err)

    close(loss, loss_ref.detach(), "loss")
    close(st["logits"].transpose(0, 1), lg_ref.detach(), "logits")
    close(torch.stack(st["alpha"], 1), al_ref.detach(), "alphas")
    for k, v in pr.items():
        close(g[k], v.grad, k)
    close(g["denc"], x.grad, "d enc")
    # the d logits the backward starts from: zero past each row's length
    valid = torch.arange(T)[:, None] < lengths[None, :]
    assert bool((st["dlogits"][~valid] == 0).all())
    assert st["dlogits"].shape == (T, enc.shape[0], V)


def test_pieces_are_what_the_reference_composes():
    """Spot checks of single pieces against their direct counterparts in oracle/ref_tf_model.py: the LSTM cell through the token
    table, the attention and the output projection of one step."""
    p, enc, formula, _, _, _, _ = _case(11, False, False)
    B = enc.shape[0]
    D, A, O = _DIMS["num_units"], _DIMS["dim_e"], _DIMS["dim_o"]
    g = torch.Generator().manual_seed(12)
    c, h, o = (torch.randn(B, n, generator=g, dtype=torch.float64) for n in (D, D, O))
    tok = formula[:, 0]
    x = torch.cat([p["embedding_table"][tok], o], 1)
    c_r, h_r = rt.lstm_cell_tf(p, x, c, h)
    _, c2, h2 = tr.lstm_pointwise(tr.gates_z(p, o, h) + tr.token_table(p)[tok], c)
    assert torch.allclose(c2, c_r, rtol=0, atol=1e-14) and torch.allclose(h2, h_r, rtol=0, atol=1e-14)
    att_img = enc @ p["att_img.kernel"]
    ctx_r, a_r = rt.attention_context(p, enc, att_img, h2)
    out2 = tr.project_h(p, h2)
    _, a, ctx = tr.attention(att_img, enc, out2[:, :A], p["att_beta"])
    assert torch.allclose(a, a_r, rtol=0, atol=1e-14) and torch.allclose(ctx, ctx_r, rtol=0, atol=1e-14)
    lg_r, (_, _, o_r), _ = rt.cell_step(p, enc, att_img, p["embedding_table"][tok], c, h, o)
    o2 = tr.output(p, ctx, out2[:, A:])
    assert torch.allclose(o2, o_r, rtol=0, atol=1e-14)
    assert torch.allclose(tr.logits(p, o2), lg_r, rtol=0, atol=1e-13)
    _, s0 = tr.initial_state(p, enc.mean(1))
    for ref, got in zip(rt.initial_state(p, enc), (s0[:, :D], s0[:, D:2 * D], s0[:, 2 * D:])):
        assert torch.allclose(got, ref, rtol=0, atol=1e-14)


# ---- the workspace layout
_SHAPES = [  # (B, T, R, C, A, D, O, E, V, ldl)
    (8, 7, 44, 512, 256, 512, 512, 80, 500, 512),
    (64, 3, 868, 512, 256, 512, 512, 80, 500, 512),
    (72, 4, 101, 512, 256, 512, 512, 80, 500, 0),
    (5, 2, 30, 1024, 1024, 640, 384, 64, 37, 64),
    (3, 9, 17, 256, 256, 96, 128, 16, 50, 56),
]


def _bytes(L, B, T, R, C, A, D, O, E, V, ldl, bf16):
    from latex_ocr_b200 import _lib
    a = _lib.TfDecArgs()
    a.B, a.T, a.R, a.C, a.A, a.D, a.O, a.E, a.V = B, T, R, C, A, D, O, E, V
    a.dt = _lib.dtype_code("bf16" if bf16 else "fp32")
    a.ldl = ldl
    a.rows_per_img = 1
    return int(L.lo_tfdec_workspace_bytes(ctypes.byref(a)))


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_workspace_layout_is_the_librarys(bf16):
    """The mirror's end offset plus a remainder that depends on B alone (the ragged decode's CTA map) is the library's workspace
    size, for two T at every shape: a region the mirror misplaces or forgets moves the end by a T-dependent amount."""
    from latex_ocr_b200 import _lib
    L = _lib.lib()
    for B, T, R, C, A, D, O, E, V, ldl in _SHAPES:
        rest = []
        for TT in (T, T + 5):
            _, end = tr.carve(B, TT, R, C, A, D, O, E, V, ldl, bf16)
            rest.append(_bytes(L, B, TT, R, C, A, D, O, E, V, ldl, bf16) - end)
        # attention_ragged_map_bytes(B): B x 16 int4 CTA map entries and B ticket counters, 256-byte aligned
        assert rest[0] == rest[1] == (B * 16 * 16 + B * 4 + 255) // 256 * 256, (B, T, rest)
