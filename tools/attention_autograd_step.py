"""Cost of training through the stand-alone Attention module at the cfg #2 shapes (bf16 storage, wgmma GEMMs, B=64, R=868,
A=C=D=512):
  (a) the single-pass step backward kernel alone (lo_attention_step_backward asked for d att1 only, which launches just that
      kernel): CUDA-event mean over --launches launches, against its byte bound (att1 and enc read, d att1 written: 3 x 56.9 MB,
      computed from the shapes) at the data sheet's 3.35 TB/s; lo_attention_backward (no d att1, att1 + enc read) beside it;
  (b) one Attention backward call (loss.backward() of a forward made outside the timed window), and one forward + backward call;
  (c) the reference's DecoderWithAttention.forward body (seq2seq_torch.py:267-320: a Python loop over 150 steps, torch LSTMCell,
      f_beta gate, fc) calling this package's Attention with a shrinking batch_size_t, forward + backward of the reference loss,
      against the fused DecoderWithAttention autograd step on the same parameters and loss.  Eval mode (no dropout) in both arms.
The card's name, power limit and max SM clock are printed with the numbers.

  python tools/attention_autograd_step.py [--launches 200] [--calls 20] [--steps 2] [--warmup 1] [--rounds 2]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import pack_padded_sequence

from latex_ocr_b200 import _lib
from latex_ocr_b200.decoder import Attention, DecoderWithAttention

B, R, A, T, V = 64, 868, 512, 150, 500


def device_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return "device: %s (%s)" % (torch.cuda.get_device_name(), q.stdout.strip() or "power limit / clock not reported")


def events_us(fn, n):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / n


def kernel_times(launches):
    """(a): µs per launch of the d att1 step kernel and of the existing step backward on the same inputs."""
    L, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr()
    g = torch.Generator(device="cuda").manual_seed(3)
    enc = (torch.randn(B, R, A, generator=g, device="cuda") * 0.5).bfloat16()
    att1 = (torch.randn(B, R, A, generator=g, device="cuda") * 0.3).bfloat16()
    att2 = torch.randn(B, A, generator=g, device="cuda") * 0.3
    wf = torch.rand(A, generator=g, device="cuda") - 0.5
    alpha = torch.softmax(torch.randn(B, R, generator=g, device="cuda"), dim=1)
    ctx = torch.randn(B, A, generator=g, device="cuda")
    dctx = torch.randn(B, A, generator=g, device="cuda")
    h, w = torch.zeros(B, A, device="cuda"), torch.zeros(A, A, dtype=torch.bfloat16, device="cuda")
    de, datt2 = torch.empty(B, R, device="cuda"), torch.empty(B, A, device="cuda")
    datt1 = torch.empty_like(att1)
    dt = _lib.LO_BF16
    work = torch.zeros(L.lo_attention_step_workspace_bytes(B, R, A, A, dt), dtype=torch.uint8, device="cuda")
    work2 = torch.zeros(L.lo_attention_workspace_bytes(B, A), dtype=torch.uint8, device="cuda")

    def step():
        L.lo_attention_step_backward(P(enc), P(att1), dt, P(h), P(att2), P(w), P(w), P(wf), P(alpha), P(ctx), P(dctx), None,
                                     None, None, None, None, None, None, None, None, P(de), P(datt2), P(datt1), B, R, A, A, A,
                                     _lib.LO_IMPL_TC, P(work), st)

    def old():
        L.lo_attention_backward(P(att1), P(enc), dt, P(att2), None, A, P(wf), P(alpha), R, P(ctx), P(dctx), A, None, 0, None, 0,
                                P(de), P(datt2), None, A, None, None, None, B, R, A, A, P(work2), st)
    n0 = _lib.launch_count()
    _lib.check(L.lo_attention_step_backward(P(enc), P(att1), dt, P(h), P(att2), P(w), P(w), P(wf), P(alpha), P(ctx), P(dctx), None,
                                            None, None, None, None, None, None, None, None, P(de), P(datt2), P(datt1), B, R, A, A, A,
                                            _lib.LO_IMPL_TC, P(work), st))
    assert _lib.launch_count() - n0 == 1
    return events_us(step, launches), events_us(old, launches), 3 * enc.numel() * 2, 2 * enc.numel() * 2


def module_times(calls):
    """(b): ms of one backward call and of one forward + backward call of Attention (bf16, wgmma)."""
    torch.manual_seed(5)
    att = Attention(A, A, A, precision="bf16")
    enc = (torch.randn(B, R, A, device="cuda") * 0.5).requires_grad_(True)
    h = torch.randn(B, A, device="cuda").requires_grad_(True)
    gc, ga = torch.randn(B, A, device="cuda"), torch.randn(B, R, device="cuda")

    def loss():
        c, a = att(enc, h)
        return (c * gc).sum() + (a * ga).sum()
    for _ in range(3):
        loss().backward()
    torch.cuda.synchronize()
    bwd = 0.0
    for _ in range(calls):
        lo = loss()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lo.backward()
        e1.record()
        torch.cuda.synchronize()
        bwd += e0.elapsed_time(e1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        loss().backward()
    e1.record()
    torch.cuda.synchronize()
    return bwd / calls, e0.elapsed_time(e1) / calls


def reference_loop(dec, encoder_out, encoded_captions, caption_lengths):
    """seq2seq_torch.py:267-320 (eval: the dropout before fc is the identity) on dec's parameter views and dec.attention."""
    Bn, C = encoder_out.size(0), encoder_out.size(-1)
    enc = encoder_out.reshape(Bn, -1, C)
    Rn = enc.size(1)
    caption_lengths, sort_ind = caption_lengths.squeeze(1).sort(dim=0, descending=True)
    sort_ind = sort_ind.to(enc.device)
    enc = enc[sort_ind]
    caps = encoded_captions[sort_ind]
    emb = F.embedding(caps, dec.embedding.weight)
    mean = enc.mean(dim=1)
    h = F.linear(mean, dec.init_h.weight, dec.init_h.bias)
    c = F.linear(mean, dec.init_c.weight, dec.init_c.bias)
    decode_lengths = (caption_lengths - 1).tolist()
    Tn = max(decode_lengths)
    preds = torch.zeros(Bn, Tn, dec.vocab_size, device=enc.device)
    alphas = torch.zeros(Bn, Tn, Rn, device=enc.device)
    ds = dec.decode_step
    for t in range(Tn):
        bt = sum(l > t for l in decode_lengths)
        ctx, alpha = dec.attention(enc[:bt], h[:bt])
        gate = torch.sigmoid(F.linear(h[:bt], dec.f_beta.weight, dec.f_beta.bias))
        h, c = torch._VF.lstm_cell(torch.cat([emb[:bt, t, :], gate * ctx], dim=1), (h[:bt], c[:bt]), ds.weight_ih, ds.weight_hh,
                                   ds.bias_ih, ds.bias_hh)
        preds[:bt, t, :] = F.linear(h, dec.fc.weight, dec.fc.bias)
        alphas[:bt, t, :] = alpha
    return preds, caps, decode_lengths, alphas, sort_ind


def reference_loss(scores, caps, decode_lengths, alphas):
    """img2seq_torch.py:147-159."""
    s = pack_padded_sequence(scores, decode_lengths, batch_first=True).data
    tg = pack_padded_sequence(caps[:, 1:], decode_lengths, batch_first=True).data
    return F.cross_entropy(s, tg) + ((1. - alphas.sum(dim=1)) ** 2).mean()


def loop_times(steps, warmup, rounds):
    """(c): ms per forward + backward of the reference loop on Attention and of the fused DecoderWithAttention."""
    torch.manual_seed(7)
    dec = DecoderWithAttention(A, A, A, V, A, precision="bf16", impl="tc")
    dec.eval()
    g = torch.Generator().manual_seed(8)
    enc = (torch.randn(B, R, A, generator=g) * 0.5).cuda().requires_grad_(True)
    caps = torch.randint(4, V, (B, T + 2), generator=g).cuda()
    lengths = torch.full((B, 1), T + 1, dtype=torch.long)
    lengths[B // 2:] = T - 20                   # ragged: half the rows stop 20 steps early

    def arm(fn):
        def step():
            dec.zero_grad(set_to_none=True)
            enc.grad = None
            reference_loss(*fn(enc, caps, lengths)[:4]).backward()
        return step
    arms = {"loop": arm(lambda *a: reference_loop(dec, *a)), "fused": arm(dec)}
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            for _ in range(warmup):
                f()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                f()
            e1.record()
            torch.cuda.synchronize()
            res[k].append(e0.elapsed_time(e1) / steps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    print(device_line())
    us, us_old, nbytes, nbytes_old = kernel_times(args.launches)
    bound = nbytes / 3.35e12 * 1e6
    print("(a) step backward kernel with d att1: %8.1f us/launch, %6.1f MB -> %7.1f GB/s; byte bound %.1f us at 3.35 TB/s (%.0f%%)"
          % (us, nbytes / 1e6, nbytes / us / 1e3, bound, 100 * bound / us))
    print("(a) lo_attention_backward (no d att1): %8.1f us/launch, %6.1f MB -> %7.1f GB/s"
          % (us_old, nbytes_old / 1e6, nbytes_old / us_old / 1e3))
    bwd, fb = module_times(args.calls)
    print("(b) Attention backward call: %.3f ms; forward + backward call: %.3f ms" % (bwd, fb))
    res = loop_times(args.steps, args.warmup, args.rounds)
    print("(c) reference loop on Attention, forward + backward: %s ms" % " ".join("%.1f" % t for t in res["loop"]))
    print("(c) fused DecoderWithAttention autograd step:       %s ms" % " ".join("%.1f" % t for t in res["fused"]))
    print("(c) loop / fused (means): %.1f" % (sum(res["loop"]) / sum(res["fused"])))


if __name__ == "__main__":
    main()
