"""Host-side restatement of the index arithmetic the tensor-core attention backward relies on (latex_ocr_b200/csrc/lo_attention.cu):
* the pair layout of the ReLU mask bits the forward kernel writes, and how a lane of `attention_bwd_mma_kernel` turns ONE 32-bit word of
  it into the four A fragments of an mma.m16n8k16 block with a shift and an AND each;
* the split of d full_att.weight (reference: autograd of seq2seq_torch.py:188-189) into the att2 term the per-step kernels accumulate and
  the att1 term the post-loop sweep adds (datt1_kernel, WACC = 2).
Pure numpy: runs without a GPU and pins the derivations next to the kernels' comments."""
import numpy as np


def _pack_pair_layout(bits):
    """bits [R][A] {0,1} -> bytes in the forward kernel's layout: byte (r, a/8) at (r/2) * 2*(A/8) + (a/8)*2 + (r&1), bit 7-(a%8)."""
    R, A = bits.shape
    MB = A // 8
    Rp = (R + 1) & ~1
    out = np.zeros(Rp * MB, np.uint8)
    for r in range(R):
        for ab in range(MB):
            v = 0
            for t in range(8):
                v |= int(bits[r, ab * 8 + t]) << (7 - t)
            out[(r >> 1) * 2 * MB + ab * 2 + (r & 1)] = v
    return out


def _byte_perm(x, y, sel):
    src = [(x >> (8 * i)) & 0xFF for i in range(4)] + [(y >> (8 * i)) & 0xFF for i in range(4)]
    return sum(src[(sel >> (4 * i)) & 0x7] << (8 * i) for i in range(4))


def test_mask_word_to_mma_fragments():
    rng = np.random.RandomState(0)
    R, A = 48, 512
    MB = A // 8
    bits = (rng.rand(R, A) < 0.5).astype(np.uint8)
    packed = _pack_pair_layout(bits)
    for row in (0, 16, 32):                                   # a 16-row stage starts on an even row: 1 KB of contiguous mask bytes
        stage = packed[(row >> 1) * 2 * MB:(row >> 1) * 2 * MB + 16 * MB]
        for w in (0, 3, 7):                                   # consumer warp = 64 attention columns
            for lane in range(32):
                g, q = lane >> 2, lane & 3
                off = q * 2 * MB + (8 * w + g) * 2            # m_off of the kernel (relative to the stage's mask bytes)
                u_lo = int(stage[off]) | (int(stage[off + 1]) << 8)
                u_hi = int(stage[off + 4 * 2 * MB]) | (int(stage[off + 4 * 2 * MB + 1]) << 8)
                mw = _byte_perm(u_lo, u_hi, 0x5140)           # [even(q) | even(q+4) | odd(q) | odd(q+4)]
                for j in range(4):
                    for ii in range(4):
                        h, rs = ii & 1, ii >> 1
                        sh = 14 - (8 * rs + 7 - (2 * j + h))
                        af = ((mw << sh) if sh >= 0 else (mw >> -sh)) & 0x40004000
                        a = 64 * w + 8 * g + 2 * j + h        # fragment row m = g + 8h of block j stands for this column
                        k = 2 * q + 8 * rs                    # fragment k index = region row of the stage
                        assert bool(af & 0x4000) == bool(bits[row + k, a])            # low half: element k
                        assert bool(af & 0x40000000) == bool(bits[row + k + 1, a])    # high half: element k + 1
                        assert af & ~0x40004000 == 0          # nothing else set: the halves are exactly bf16 0.0 or 2.0


def test_full_att_weight_gradient_split():
    """d w[a] = sum_{b,r,t} de[b,t,r] relu(x[b,r,a] + a2[t,b,a])
             = sum_{b,r} x[b,r,a] acc[b,r,a]                      (sweep over att1: acc = sum_t de * on)
             + sum_{t,b} a2[t,b,a] S[t,b,a]                       (per-step kernels: S = sum_r de * on = datt2 / w)"""
    rng = np.random.RandomState(1)
    B, R, A, T = 3, 7, 16, 5
    x = rng.randn(B, R, A)
    a2 = rng.randn(T, B, A)
    de = rng.randn(B, T, R)
    pre = x[:, None] + a2.transpose(1, 0, 2)[:, :, None]      # [B,T,R,A]
    on = pre > 0
    want = (de[..., None] * np.maximum(pre, 0)).sum(axis=(0, 1, 2))
    acc = (de[..., None] * on).sum(axis=1)                    # [B,R,A]
    S = (de[..., None] * on).sum(axis=2)                      # [B,T,A]
    got = (x * acc).sum(axis=(0, 1)) + (a2.transpose(1, 0, 2) * S).sum(axis=(0, 1))
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_hi_lo_split_keeps_fp32_products():
    """The B operands of both contractions are fp32 values split into a bf16 high part and a bf16 residual: with bf16 A operands the
    products are exact in fp32 and hi + lo carries 16 mantissa bits (relative error <= 2^-16) instead of bf16's 8."""
    import torch
    v = torch.randn(4096, dtype=torch.float32) * torch.logspace(-6, 2, 4096)
    hi = v.bfloat16()
    lo = (v - hi.float()).bfloat16()
    rec = hi.float() + lo.float()
    rel = ((rec - v).abs() / v.abs().clamp_min(1e-30)).max().item()
    assert rel <= 2.0 ** -16
    assert ((hi.float() - v).abs() / v.abs().clamp_min(1e-30)).max().item() > 2.0 ** -10      # what a single bf16 would lose

