"""Cost of scheduled sampling at the cfg #2 workload (bf16, B=64, 128x512 images, T=150, V=500, dropout on, p = 0.25):
  (a) the fused Img2SeqModel.getLoss, teacher forcing (eager);
  (b) the fused getLoss with set_sampling_prob(0.25), eager and replayed as a CUDA graph;
  (c) autograd: model.decoder(..., sampling_prob=0.25) + the reference loss (img2seq_torch.py:147-159) + two torch.optim.Adam;
  (d) the per-step Python loop of INTEGRATION.md §1 (torch LSTM cell, f_beta gate, fc, scheduled sampling) on the CUDA
      Attention, forward + backward of the reference loss + two torch.optim.Adam, --loop-steps steps after one warm-up step;
  (e) the head GEMM the sampling mode adds to every step: lo_gemm of 64 bf16 rows x fc.weight (N = 500, K = 512), rows T*D apart,
      fp32 out, on the mma.sync kernel the decoder's step loop uses — CUDA-event mean over --launches back-to-back launches.
Times are CUDA-event means over the timed steps after warm-up.  The card's name, power limit and max SM clock are printed with
the numbers.

  python tools/scheduled_sampling_step.py [--steps 10] [--warmup 3] [--loop-steps 2] [--launches 300]
"""
import argparse
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch
import torch.nn as nn
import torch.nn.functional as F

import bench_support as bs
from attention_autograd_step import device_line, events_us, reference_loss
from autograd_step import B, H, T, V, W, make_model, reference_step, time_ms
from latex_ocr_b200 import _lib

P_SAMPLE = 0.25


def sampled_reference_step(model, opt_e, opt_d, crit, img, formula):
    """(c): reference_step with the fused decoder asked for scheduled sampling."""
    dec = model.decoder
    fwd = dec.forward
    dec.forward = lambda *a: fwd(*a, sampling_prob=P_SAMPLE)
    try:
        return reference_step(model, opt_e, opt_d, crit, img, formula)
    finally:
        del dec.forward


def integration_loop_step(model, opt_e, opt_d, img, formula):
    """(d): INTEGRATION.md §1's loop (seq2seq_torch.py:267-320 edited for scheduled sampling) + reference loss + Adam."""
    dec = model.decoder
    encoder_out = model.encoder(img)
    Bn, C = encoder_out.size(0), encoder_out.size(-1)
    enc = encoder_out.reshape(Bn, -1, C)
    Rn = enc.size(1)
    caption_lengths, sort_ind = torch.LongTensor([[len(i)] for i in formula]).squeeze(1).sort(dim=0, descending=True)
    sort_ind = sort_ind.to(enc.device)
    enc = enc[sort_ind]
    caps = formula[sort_ind]
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
        tok = caps[:bt, t] if random.random() > P_SAMPLE else preds[:bt, t - 1].argmax(-1) if t else caps[:bt, 0]
        x = torch.cat([F.embedding(tok, dec.embedding.weight), gate * ctx], dim=1)
        h, c = torch._VF.lstm_cell(x, (h[:bt], c[:bt]), ds.weight_ih, ds.weight_hh, ds.bias_ih, ds.bias_hh)
        preds[:bt, t] = F.linear(F.dropout(h, 0.5, dec.training), dec.fc.weight, dec.fc.bias)
        alphas[:bt, t] = alpha
    loss = reference_loss(preds, caps, decode_lengths, alphas)
    opt_d.zero_grad()
    opt_e.zero_grad()
    loss.backward()
    opt_d.step()
    opt_e.step()
    return -loss.item()


def head_gemm_us(launches):
    """(e): µs per launch of the per-step head GEMM at the cfg #2 shapes."""
    L, Pt, st = _lib.lib(), _lib.ptr, _lib.stream_ptr()
    D, ldl = 512, (V + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(7)
    hd = (torch.randn(B, T, D, generator=g, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(V, D, generator=g, device="cuda") * 0.05).bfloat16()
    bias = torch.zeros(V, device="cuda")
    logits = torch.empty(B, T, ldl, device="cuda")

    def launch():
        _lib.check(L.lo_gemm(Pt(hd), _lib.LO_BF16, Pt(w), _lib.LO_BF16, Pt(logits), _lib.LO_F32, B, V, D, T * D, 1, 1, D, T * ldl,
                             1, 0, 0, 0, Pt(bias), 0, 0, _lib.LO_IMPL_TC, st))
    return events_us(launch, launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop-steps", type=int, default=2)
    ap.add_argument("--launches", type=int, default=300)
    args = ap.parse_args()
    print(device_line())
    random.seed(0)
    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.cuda(), formula.cuda()
    res = {}
    fused = make_model(False)
    res["a"] = time_ms(lambda: fused.getLoss(img, formula, None, None), args.steps, args.warmup)
    fused.set_sampling_prob(P_SAMPLE)
    res["b eager"] = time_ms(lambda: fused.getLoss(img, formula, None, None), args.steps, args.warmup)
    del fused
    graphed = make_model(True)
    graphed.set_sampling_prob(P_SAMPLE)
    res["b graph"] = time_ms(lambda: graphed.getLoss(img, formula, None, None), args.steps, args.warmup)
    del graphed
    auto = make_model(False)
    opt_e = torch.optim.Adam(auto.encoder.parameters(), lr=1e-3)
    opt_d = torch.optim.Adam(auto.decoder.parameters(), lr=1e-3)
    crit = nn.CrossEntropyLoss()
    res["c"] = time_ms(lambda: sampled_reference_step(auto, opt_e, opt_d, crit, img, formula), args.steps, args.warmup)
    res["d"] = time_ms(lambda: integration_loop_step(auto, opt_e, opt_d, img, formula), args.loop_steps, 1)
    res["e"] = head_gemm_us(args.launches)
    names = {"a": "fused getLoss, teacher forcing, eager", "b eager": "fused getLoss, p = 0.25, eager",
             "b graph": "fused getLoss, p = 0.25, CUDA graph",
             "c": "autograd dec(..., sampling_prob=0.25) + reference loss + Adam",
             "d": "INTEGRATION.md loop (p = 0.25) + reference loss + Adam"}
    for k in ("a", "b eager", "b graph", "c", "d"):
        print("(%-7s) %-62s %8.2f ms/step" % (k, names[k], res[k]))
    print("(e      ) per-step head GEMM (64 x 500 x 512, bf16 mma.sync)                 %8.2f us/launch" % res["e"])
    print("(b eager) / (a) = %.3f ; (d) / (b eager) = %.1f" % (res["b eager"] / res["a"], res["d"] / res["b eager"]))


if __name__ == "__main__":
    main()
