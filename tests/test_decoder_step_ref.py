"""CPU: the per-step float64 restatement of the decoder (tests/decoder_step_ref.py), chained over T steps, reproduces the hoisted
forward and the hand-derived backward of oracle/ref_model.py.  tests/test_gpu_decoder_steps.py compares the kernels with the
pieces of that restatement one step at a time; this test is what ties those pieces to the reference."""
import pytest
import torch

import decoder_step_ref as ds
from oracle import ref_model as rm


def _case(dropout, seed):
    B, R, C, D, E, V, T = 3, 7, 16, 12, 8, 13, 5
    _, p = rm.init_params(V, seed=seed, attention_dim=C, embed_dim=E, decoder_dim=D, encoder_dim=C, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed + 1)
    for k in p:                     # biases and fc away from their zero / small init, so that every term is exercised
        p[k] = p[k] + 0.2 * torch.randn(p[k].shape, generator=g, dtype=torch.float64)
    enc = torch.randn(B, R, C, generator=g, dtype=torch.float64)
    caps = torch.randint(0, V, (B, T + 1), generator=g)
    mult = None
    if dropout:
        mult = (torch.rand(B, T, D, generator=g, dtype=torch.float64) >= 0.5).double() * 2.0
    return p, enc, caps, T, mult


@pytest.mark.parametrize("dropout", [False, True], ids=["no-dropout", "dropout"])
def test_chained_steps_match_the_reference(dropout):
    p, enc, caps, T, mult = _case(dropout, seed=5 + dropout)
    s = rm.decoder_forward_saved(p, enc, caps, T, dropout_mask=mult)
    loss_ref, g_ref, denc_ref = rm.decoder_backward_manual(p, s)
    loss, st, g = ds.chained(p, enc, caps, T, mult)

    def close(a, b, what):
        err = (a - b).abs().max().item()
        assert err <= 1e-12 * max(1.0, b.abs().max().item()), (what, err)

    close(loss, loss_ref, "loss")
    close(st["logits"], s["logits"], "logits")
    close(st["alphas"], s["alphas"], "alphas")
    for k in ("h", "c", "i", "f", "g", "o", "ctx", "att2"):
        for t in range(T):
            close(st[k][t], s[k][t], "%s[%d]" % (k, t))
    ref = ds.as_reference_grads(p, g)
    for k, v in ref.items():
        close(v, g_ref[k], k)
    close(g["denc"], denc_ref, "d encoder_out")
    assert abs(g_ref["attention.full_att.bias"].item()) < 1e-12      # sum_r de = 0: the kernels write 0 for it


def test_pieces_are_what_the_reference_composes():
    """Spot checks of single pieces where the reference has a direct counterpart: the attention and the LSTM cell of
    oracle/ref_model.py's forward, the cross entropy and its gradient of torch's log_softmax."""
    p, enc, caps, T, _ = _case(False, seed=11)
    C = enc.shape[2]
    A = p["attention.encoder_att.weight"].shape[0]
    h = torch.randn(enc.shape[0], p["init_h.weight"].shape[0], dtype=torch.float64)
    c = torch.randn_like(h)
    att1 = ds.linear(enc, p["attention.encoder_att.weight"], p["attention.encoder_att.bias"])[0]
    out1 = ds.project(p, h)
    gate = torch.sigmoid(out1[:, A:A + C])
    _, alpha, ctx, gctx = ds.attention(att1, enc, out1[:, :A], p["attention.full_att.weight"].reshape(-1), gate)
    ctx_r, alpha_r = rm.attention_forward(p, enc, h, att1)
    assert torch.allclose(alpha, alpha_r, rtol=0, atol=1e-14) and torch.allclose(ctx, ctx_r, rtol=0, atol=1e-14)
    x = torch.cat([p["embedding.weight"][caps[:, 0]], gctx], 1)
    h_r, c_r = rm.lstm_cell(p, x, h, c)
    *_, c2, h2 = ds.cell(p, gctx, ds.proj_table(p, C)[caps[:, 0]], out1[:, A + C:], c)
    assert torch.allclose(h2, h_r, rtol=0, atol=1e-14) and torch.allclose(c2, c_r, rtol=0, atol=1e-14)
    logits = torch.randn(6, 13, dtype=torch.float64)
    tg = torch.randint(0, 13, (6,))
    row, d = ds.cross_entropy(logits, tg, 1.0 / 6)
    lsm = torch.log_softmax(logits, -1)
    assert torch.allclose(row, -lsm.gather(-1, tg[:, None])[:, 0], rtol=0, atol=1e-13)
    lt = logits.clone().requires_grad_(True)
    torch.nn.functional.cross_entropy(lt, tg).backward()
    assert torch.allclose(d, lt.grad, rtol=0, atol=1e-15)
