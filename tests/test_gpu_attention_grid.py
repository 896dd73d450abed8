"""-m gpu: the launch geometry of the attention forward pipe kernel and the tensor-core backward changes no bit.

Option att_cluster picks how the splits of a batch row meet: 2 always as a thread-block cluster (combine through distributed
shared memory), 1 (default) without a cluster whenever the cluster-free grid is one resident wave (the last CTA of a row combines
the partials from global memory).  Both combines add the splits in the same order with the same operations, so every output must
be equal bit for bit, not merely close."""
import ctypes

import pytest
import torch

from util import build_model

pytestmark = pytest.mark.gpu

P = None


def _L():
    global P
    from latex_ocr_b200 import _lib
    P = _lib.ptr
    return _lib, _lib.lib()


def _fwd_inputs(B, R, A, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    O1 = 2 * A + 64
    att1 = (torch.randn(B, R, A, device="cuda", generator=g) * 0.5).to(dtype)
    enc = torch.randn(B, R, A, device="cuda", generator=g).to(dtype)
    o1 = torch.randn(B, O1, device="cuda", generator=g) * 0.5          # att2 | gate pre-activation | unused
    wf = torch.randn(A, device="cuda", generator=g) * 0.2
    return att1, enc, o1, wf, O1


def _forward(att1, enc, o1, wf, O1, mask):
    """One stand-alone forward launch; returns alpha, ctx, gate (after the sigmoid), gctx and the mask bits."""
    _lib, L = _L()
    B, R, A = att1.shape
    dt = _lib.dt_of(enc)
    o1 = o1.clone()                                  # the gate is finalised in place
    alpha = torch.full((B, R), float("nan"), device="cuda")
    ctx = torch.full((B, A), float("nan"), device="cuda")
    gctx = torch.full((B, A), float("nan"), device="cuda")
    work = torch.zeros(L.lo_attention_workspace_bytes(B, A), dtype=torch.uint8, device="cuda")
    gate = ctypes.c_void_p(o1.data_ptr() + A * 4)
    if mask:
        bits = torch.zeros(B, (R + 1) // 2 * 2, A // 8, dtype=torch.uint8, device="cuda")
        _lib.check(L.lo_attention_forward_mask(P(att1), P(enc), dt, P(o1), O1, P(wf), P(alpha), R, P(ctx), gate, O1, P(gctx), P(bits),
                                               B, R, A, A, P(work), _lib.stream_ptr()))
    else:
        bits = None
        _lib.check(L.lo_attention_forward(P(att1), P(enc), dt, P(o1), O1, P(wf), P(alpha), R, P(ctx), gate, O1, P(gctx),
                                          B, R, A, A, P(work), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return [t for t in (alpha, ctx, o1[:, A:2 * A].clone(), gctx, bits) if t is not None]


@pytest.mark.parametrize("dtype,mask", [(torch.bfloat16, True), (torch.float32, False)], ids=["bf16-mask", "fp32"])
@pytest.mark.parametrize("B,R", [(64, 868), (40, 868), (5, 101)])
def test_forward_grid_choice_is_bit_identical(dtype, mask, B, R):
    _lib, _ = _L()
    A = 512
    ins = _fwd_inputs(B, R, A, dtype, seed=11 * B + R)
    out = {}
    for val in (2, 1):
        with _lib.option(att_cluster=val):
            out[val] = _forward(*ins, mask)
    for name, a, b in zip(("alpha", "ctx", "gate", "gctx", "mask bits"), out[2], out[1]):
        assert torch.equal(a, b), name
    assert torch.isfinite(out[1][0]).all() and torch.isfinite(out[1][1]).all()


def test_backward_grid_choice_is_bit_identical_over_steps():
    """The tensor-core backward (bf16, mask bits, A = C = 512) over three consecutive steps: de, d att2, d gate and the d w_full
    partial that the steps accumulate."""
    _lib, L = _L()
    B, R, A = 64, 868, 512
    att1, enc, o1, wf, O1 = _fwd_inputs(B, R, A, torch.bfloat16, seed=5)
    g = torch.Generator(device="cuda").manual_seed(6)
    steps = []
    for s in range(3):
        o1s = o1 + 0.1 * s
        alpha, ctx, gate, _, bits = _forward(att1, enc, o1s, wf, O1, True)
        o1f = o1s.clone()
        o1f[:, A:2 * A] = gate                       # the backward reads the gate after the sigmoid
        dgctx = torch.randn(B, A, device="cuda", generator=g)
        dreg = torch.randn(B, R, device="cuda", generator=g) * 1e-3
        sreg = torch.randn(B, device="cuda", generator=g) * 1e-3
        steps.append((o1f, alpha, ctx, dgctx, dreg, sreg, bits))
    out = {}
    for val in (2, 1):
        with _lib.option(att_cluster=val):
            dwf = torch.zeros(B, A, device="cuda")
            res = []
            for o1f, alpha, ctx, dgctx, dreg, sreg, bits in steps:
                de = torch.full((B, R), float("nan"), device="cuda")
                dcat = torch.full((B, 2 * A), float("nan"), device="cuda")
                work = torch.zeros(L.lo_attention_workspace_bytes(B, A), dtype=torch.uint8, device="cuda")
                _lib.check(L.lo_attention_backward(P(att1), P(enc), _lib.LO_BF16, P(o1f), ctypes.c_void_p(o1f.data_ptr() + A * 4), O1,
                                                   P(wf), P(alpha), R, P(ctx), P(dgctx), A, P(dreg), R, P(sreg), 1, P(de), P(dcat),
                                                   ctypes.c_void_p(dcat.data_ptr() + A * 4), 2 * A, None, P(dwf), P(bits), B, R, A, A,
                                                   P(work), _lib.stream_ptr()))
                torch.cuda.synchronize()
                res += [de, dcat[:, :A].clone(), dcat[:, A:].clone(), dwf.clone()]
            out[val] = res
    for i, (a, b) in enumerate(zip(out[2], out[1])):
        assert torch.equal(a, b), ("step", i // 4, ("de", "datt2", "dgate", "dwf_part")[i % 4])
    assert torch.isfinite(out[1][-1]).all()


def _train_case(B, H, W, V=60, T=5, seed=21):
    from oracle import ref_model as rm
    pe, pd = rm.init_params(V, seed=seed)
    img, formula = rm.synthetic_batch(B, H, W, V, T, T, seed=seed + 1)
    return V, pe, pd, img, formula


def _params_after_steps(V, pe, pd, img, formula, graph, steps):
    m = build_model(V, pe, pd, "bf16", impl="tc", graph=graph)
    for _ in range(steps):
        m.train_step(img, formula)
    torch.cuda.synchronize()
    return [t.clone() for s_ in (m.encoder.store, m.decoder.store) for t in (s_.grad, s_.master)]


def test_train_step_grid_choice_is_bit_identical():
    """One full train step at the bench's image size (B = 64, 128 x 512: R = 868 regions) in deterministic mode: the gradients and
    every parameter after Adam.  The step also consumes the bf16 mirrors of gctx and d att2 that only the decoder asks for."""
    _lib, _ = _L()
    case = _train_case(64, 128, 512)
    out = {}
    with _lib.option(deterministic=1):
        for val in (2, 1):
            with _lib.option(att_cluster=val):
                out[val] = _params_after_steps(*case, graph=False, steps=1)
    for i, (a, b) in enumerate(zip(out[2], out[1])):
        assert torch.equal(a, b), ("encoder", "decoder")[i // 2] + (" grad", " parameters")[i % 2]


def test_graph_replay_grid_choice_is_bit_identical():
    """The grid choice is made once per kernel and shared memory size and cached, so capturing a train step records the same
    launches eager execution makes: two captured-and-replayed steps (deterministic mode) give the bits of the cluster launches."""
    _lib, _ = _L()
    case = _train_case(64, 128, 512, seed=31)
    out = {}
    with _lib.option(deterministic=1):
        for val in (2, 1):
            with _lib.option(att_cluster=val):
                out[val] = _params_after_steps(*case, graph=True, steps=2)
    for i, (a, b) in enumerate(zip(out[2], out[1])):
        assert torch.equal(a, b), ("encoder", "decoder")[i // 2] + (" grad", " parameters")[i % 2]


@pytest.mark.parametrize("precision,impl", [("fp32", "simt"), ("bf16", "tc")])
def test_beam_layout_grid_choice_is_bit_identical(precision, impl):
    """Beam search: rows_per_img consecutive rows attend over one image."""
    from latex_ocr_b200 import decode
    from oracle import ref_model as rm
    _lib, _ = _L()
    V = 30
    pe, pd = rm.init_params(V, seed=8)
    g = torch.Generator().manual_seed(8)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    img, _ = rm.synthetic_batch(4, 32, 80, V, 3, 5, seed=9)
    out = {}
    for val in (2, 1):
        with _lib.option(att_cluster=val):
            m = build_model(V, pe, pd, precision, impl=impl)
            out[val] = decode.beam_decode(m, img, start_id=V - 2, end_id=5, beam_size=3, max_length_formula=8)
    assert torch.equal(out[2][0], out[1][0])
    assert torch.equal(out[2][1], out[1][1])
