"""The element-wise checks of the float64 step tests (tests/test_gpu_decoder_steps.py, tests/test_gpu_lstmseq_steps.py): the
checker that records the worst |y - ref| / bound per quantity, and the bounds of an LSTM cell and its backward derived in the
docstring of tests/test_gpu_decoder_steps.py."""
import torch

SENTINEL = -1536.0                  # exact in bf16 and fp32, never produced by the data here
ACC = 2.0 ** -16                    # fp32 GEMM / reduction outputs: |y - ref| <= ACC x the sum of the magnitudes of the terms
ULPS = 2.0 ** -21                   # a few fp32 ulps of a value <= 1


def rn(x):
    """x rounded to bf16, as float64."""
    return x.bfloat16().double()


def half_ulp_bf16(ref):
    _, e = torch.frexp(ref)
    return torch.where(ref != 0, torch.ldexp(torch.full_like(ref, 0.5), e - 8), torch.zeros_like(ref))


def bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


class Checker:
    def __init__(self, tag):
        self.tag = tag
        self.worst = {}

    def bound(self, name, y, ref, bound):
        """|y - ref| <= bound element-wise (NaN fails); records the worst ratio."""
        d = (y.double() - ref).abs()
        bound = torch.broadcast_to(torch.as_tensor(bound, dtype=torch.float64, device=d.device), d.shape)
        ok = d <= bound
        if not bool(ok.all()):
            bad = (~ok).nonzero()
            i = tuple(bad[0].tolist())
            raise AssertionError("%s %s: %d of %d elements outside the bound; first at %s: got %r, float64 %r, bound %.3g"
                                 % (self.tag, name, bad.shape[0], y.numel(), i, y[i].item(), ref[i].item(), bound[i].item()))
        r = torch.where(bound > 0, d / bound.clamp_min(1e-300), torch.zeros_like(d)).max().item() if d.numel() else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)

    def gemm(self, name, y, ref, S):
        self.bound(name, y, ref, ACC * S)

    def attn(self, name, y, ref):
        """The attention kernels' rule: 1e-5 of max |ref| plus 2e-8."""
        self.bound(name, y, ref, torch.full_like(ref, 1e-5 * ref.abs().max().item() + 2e-8))

    def exact(self, name, y, ref):
        assert torch.equal(bits(y), bits(ref.to(y.dtype))), "%s %s: not bit for bit" % (self.tag, name)

    def value(self, name, y, v):
        assert bool((y == v).all()), "%s %s: expected every element to be %r" % (self.tag, name, v)


def check_gates(ck, gates, pre, e_pre):
    """The post-activation gates [..][4H] (i, f, g, o) from the pre-activations and their allowance: sigmoid is 1/4-Lipschitz,
    tanh 1-Lipschitz, plus a few ulps."""
    H = gates.shape[-1] // 4
    for q, (fn, lip) in enumerate(((torch.sigmoid, 0.25), (torch.sigmoid, 0.25), (torch.tanh, 1.0), (torch.sigmoid, 0.25))):
        sl = slice(q * H, (q + 1) * H)
        ck.bound("gates", gates[..., sl], fn(pre[..., sl]), lip * e_pre[..., sl] + ULPS)


def check_cell(ck, c_new, h_new, i, f, g, o, c_prev):
    """c and h from the kernel's own gates and c_prev (float64): only their roundings remain."""
    ck.bound("c", c_new, f * c_prev + i * g, 2.0 ** -22 * ((f * c_prev).abs() + (i * g).abs()) + 1e-38)
    href = o * torch.tanh(c_new.double())
    ck.bound("h", h_new, href, 2.0 ** -21 * href.abs() + 1e-38)


def cell_backward_bounds(e_dc, e_dh, dc, dh, dct, i, f, g, o, th, cp, dG):
    """(bound on the four gate gradients [..][4H], allowance E of dct) of the cell backward: dc the float64 carried d c with its
    allowance e_dc, dh with its allowance e_dh, th = tanh of the kernel's c, cp the kernel's c_prev."""
    e_dct = (e_dc + e_dh * (o * (1 - th * th)).abs() + (dh * o).abs() * (2 * th.abs() * 2.0 ** -22 * th.abs() + 2.0 ** -23)
             + 2.0 ** -22 * (dc.abs() + (dh * o * (1 - th * th)).abs()))
    bnd = torch.cat([e_dct * (g * i * (1 - i)).abs(), e_dct * (cp * f * (1 - f)).abs(),
                     e_dct * (i * (1 - g * g)).abs() + (dct * i).abs() * 2.0 ** -23,
                     e_dh * (th * o * (1 - o)).abs() + (dh * o * (1 - o)).abs() * 2.0 ** -22 * th.abs()], -1) + ULPS * dG.abs()
    return bnd + 1e-38, e_dct
