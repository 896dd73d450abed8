"""-m gpu: the L2 residency budget of the attention launches (option att_l2_keep_mb) changes where the bytes come from, never a bit.

The budget only picks the cache hint of each ring stage's bulk copies (kept: evict_normal, streamed: evict_first); the row partition,
the ring and every sum stay as they are.  So each output must be equal bit for bit for budget 0 (nothing kept), the default, a budget
above the launch's bytes (clamped to the L2: everything that may be kept is) and an odd value."""
import ctypes

import pytest
import torch

from test_gpu_attention_grid import _forward, _fwd_inputs, _params_after_steps, _train_case
from util import build_model

pytestmark = pytest.mark.gpu


def _lib_L():
    from latex_ocr_b200 import _lib
    return _lib, _lib.lib()


def _budgets():
    _lib, L = _lib_L()
    default = L.lo_get_option(b"att_l2_keep_mb")
    assert default > 0
    return [0, default, 4096, 13]


def _backward_steps(att1, enc, o1, wf, O1, steps):
    """the tensor-core backward (bf16, mask bits, A = C = 512) over consecutive steps: de, d att2, d gate, the d w_full partial"""
    _lib, L = _lib_L()
    P = _lib.ptr
    B, R, A = att1.shape
    dwf = torch.zeros(B, A, device="cuda")
    res = []
    for o1f, alpha, ctx, dgctx, dreg, sreg, bits in steps:
        de = torch.full((B, R), float("nan"), device="cuda")
        dcat = torch.full((B, 2 * A), float("nan"), device="cuda")
        dctx = torch.full((B, A), float("nan"), device="cuda")
        work = torch.zeros(L.lo_attention_workspace_bytes(B, A), dtype=torch.uint8, device="cuda")
        _lib.check(L.lo_attention_backward(P(att1), P(enc), _lib.LO_BF16, P(o1f), ctypes.c_void_p(o1f.data_ptr() + A * 4), O1,
                                           P(wf), P(alpha), R, P(ctx), P(dgctx), A, P(dreg), R, P(sreg), 1, P(de), P(dcat),
                                           ctypes.c_void_p(dcat.data_ptr() + A * 4), 2 * A, P(dctx), P(dwf), P(bits), B, R, A, A,
                                           P(work), _lib.stream_ptr()))
        torch.cuda.synchronize()
        res += [de, dcat[:, :A].clone(), dcat[:, A:].clone(), dctx, dwf.clone()]
    return res


@pytest.mark.parametrize("B,R", [(64, 868), (40, 101)])
def test_attention_launches_are_bit_identical_for_every_budget(B, R):
    """forward (bf16 with mask bits) and, on its outputs, the tensor-core backward over three steps"""
    _lib, _ = _lib_L()
    A = 512
    att1, enc, o1, wf, O1 = _fwd_inputs(B, R, A, torch.bfloat16, seed=7 * B + R)
    g = torch.Generator(device="cuda").manual_seed(B)
    grads = [(torch.randn(B, A, device="cuda", generator=g), torch.randn(B, R, device="cuda", generator=g) * 1e-3,
              torch.randn(B, device="cuda", generator=g) * 1e-3) for _ in range(3)]
    out = {}
    for kb in _budgets():
        with _lib.option(att_l2_keep_mb=kb):
            fwd, steps = [], []
            for s in range(3):
                o1s = o1 + 0.1 * s
                alpha, ctx, gate, gctx, bits = _forward(att1, enc, o1s, wf, O1, True)
                fwd += [alpha, ctx, gate, gctx, bits]
                o1f = o1s.clone()
                o1f[:, A:2 * A] = gate                   # the backward reads the gate after the sigmoid
                steps.append((o1f, alpha, ctx) + grads[s] + (bits,))
            out[kb] = (fwd, _backward_steps(att1, enc, o1, wf, O1, steps))
    ref = out[0]
    fnames, bnames = ("alpha", "ctx", "gate", "gctx", "mask bits"), ("de", "datt2", "dgate", "dctx", "dwf_part")
    for kb, (fwd, bwd) in out.items():
        for i, (a, b) in enumerate(zip(ref[0], fwd)):
            assert torch.equal(a, b), (kb, "forward step", i // 5, fnames[i % 5])
        for i, (a, b) in enumerate(zip(ref[1], bwd)):
            assert torch.equal(a, b), (kb, "backward step", i // 5, bnames[i % 5])
    assert torch.isfinite(ref[1][-1]).all() and torch.isfinite(ref[0][1]).all()


def test_train_step_is_bit_identical_for_every_budget():
    """one deterministic train step at the bench's image size (B = 64, 128 x 512: R = 868): gradients and parameters after Adam"""
    _lib, _ = _lib_L()
    case = _train_case(64, 128, 512, seed=41)
    out = {}
    with _lib.option(deterministic=1):
        for kb in _budgets():
            with _lib.option(att_l2_keep_mb=kb):
                out[kb] = _params_after_steps(*case, graph=False, steps=1)
    for kb, res in out.items():
        for i, (a, b) in enumerate(zip(out[0], res)):
            assert torch.equal(a, b), (kb, ("encoder", "decoder")[i // 2] + (" grad", " parameters")[i % 2])


def test_graph_replay_is_bit_identical_for_every_budget():
    """the keep share is a launch argument, so a captured step records it: two replayed steps give the budget-0 replay's bits"""
    _lib, _ = _lib_L()
    case = _train_case(64, 128, 512, seed=43)
    with _lib.option(deterministic=1):
        with _lib.option(att_l2_keep_mb=0):
            ref = _params_after_steps(*case, graph=True, steps=2)
        for kb in _budgets()[1:]:
            with _lib.option(att_l2_keep_mb=kb):
                res = _params_after_steps(*case, graph=True, steps=2)
            for i, (a, b) in enumerate(zip(ref, res)):
                assert torch.equal(a, b), (kb, ("encoder", "decoder")[i // 2] + (" grad", " parameters")[i % 2])


def test_predict_images_tokens_are_identical_for_every_budget():
    """greedy and beam decoding of images of different sizes (ragged launch; beam: several rows attend over one image)"""
    from oracle import ref_model as rm
    _lib, _ = _lib_L()
    V = 30
    pe, pd = rm.init_params(V, seed=12)
    g = torch.Generator().manual_seed(12)
    pd["fc.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 0.5
    pd["embedding.weight"] = (torch.rand(V, 512, generator=g) * 2 - 1) * 1.0
    imgs = []
    for k, (H, W) in enumerate(((32, 64), (48, 96), (32, 200), (64, 320))):
        imgs += list(rm.synthetic_batch(2, H, W, V, 3, 5, seed=50 + k)[0].to(torch.uint8))
    m = build_model(V, pe, pd, "bf16", impl="tc")
    out = {}
    for kb in _budgets():
        with _lib.option(att_l2_keep_mb=kb):
            out[kb] = [m.predict_images(imgs, decoding=d, beam_size=k) for d, k in (("greedy", 1), ("beam_search", 3))]
    for kb, res in out.items():
        assert res == out[0], kb
