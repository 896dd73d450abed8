"""Cost of self-critical training at the cfg #2 workload (bf16, B=64, 128x512 images, T=150, V=500, dropout on, tau = 1):
  (a) the fused Img2SeqModel.getLoss, cross-entropy (eager);
  (b) the fused getLoss with set_self_critical(1.0), eager and replayed as a CUDA graph;
  (c) the autograd route: encoder, greedy rollout under no_grad, decoder(..., sampling_prob=1, sampling_temperature=1),
      scst.rewards, the policy-gradient loss in plain torch, backward, two torch.optim.Adam;
  (d) the sampling pointwise kernel against the argmax one: a whole no-grad decoder forward at p = 1 (eval mode, all 150 steps)
      with and without the temperature; the difference over T is the added cost per step.
Times are CUDA-event means over the timed steps after warm-up.  The card's name, power limit and max SM clock are printed with
the numbers.

  python tools/scst_step.py [--steps 10] [--warmup 3]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch
import torch.nn.functional as F

import bench_support as bs
from attention_autograd_step import device_line
from autograd_step import B, H, T, V, W, make_model, time_ms
from latex_ocr_b200 import scst

TAU = 1.0


def autograd_step(model, opt_e, opt_d, img, formula, end_id):
    """(c): the SCST recipe of INTEGRATION.md §1 through autograd."""
    dec = model.decoder
    N, L = formula.shape
    lens = torch.full((N, 1), L, dtype=torch.long)
    enc = model.encoder(img)
    with torch.no_grad():
        dec.eval()
        dec(enc.detach(), formula, lens, sampling_prob=1.0)
        greedy = dec.last_fed_tokens.clone()
        dec.train()
    preds, caps, _, _, _ = dec(enc, formula, lens, sampling_prob=1.0, sampling_temperature=TAU)
    fed = dec.last_fed_tokens
    _, _, adv, n_len = scst.rewards(fed, caps, end_id, greedy=greedy)
    Tn = preds.shape[1]
    lp = F.log_softmax(preds / TAU, dim=-1)[:, :Tn - 1].gather(2, fed[:, 1:].unsqueeze(2)).squeeze(2)
    act = (torch.arange(1, Tn, device=preds.device)[None, :] <= n_len.long()[:, None]).float()
    loss = -(adv[:, None] * lp * act).sum() / N
    opt_d.zero_grad()
    opt_e.zero_grad()
    loss.backward()
    opt_d.step()
    opt_e.step()
    return -loss.item()


def forward_ms(dec, enc, formula, lens, tau, steps, warmup):
    """(d): ms per no-grad decoder forward at p = 1."""
    def run():
        with torch.no_grad():
            dec(enc, formula, lens, sampling_prob=1.0, sampling_temperature=tau)
    return time_ms(run, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print(device_line())
    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.cuda(), formula.cuda()
    res = {}
    fused = make_model(False)
    end_id = fused._end_id()
    res["a"] = time_ms(lambda: fused.getLoss(img, formula, None, None), args.steps, args.warmup)
    fused.set_self_critical(TAU)
    res["b eager"] = time_ms(lambda: fused.getLoss(img, formula, None, None), args.steps, args.warmup)
    print("fused SCST stats after the eager steps [L, mean r_sample, mean r_greedy, mean n_b]:",
          [round(x, 4) for x in fused.train_step(img, formula, sync=True).tolist()])
    del fused
    graphed = make_model(True)
    graphed.set_self_critical(TAU)
    res["b graph"] = time_ms(lambda: graphed.getLoss(img, formula, None, None), args.steps, args.warmup)
    del graphed
    auto = make_model(False)
    opt_e = torch.optim.Adam(auto.encoder.parameters(), lr=1e-3)
    opt_d = torch.optim.Adam(auto.decoder.parameters(), lr=1e-3)
    res["c"] = time_ms(lambda: autograd_step(auto, opt_e, opt_d, img, formula, end_id), args.steps, args.warmup)
    dec = auto.decoder
    dec.eval()
    with torch.no_grad():
        enc = auto.encoder(img)
    lens = torch.full((B, 1), formula.shape[1], dtype=torch.long)
    res["d argmax"] = forward_ms(dec, enc, formula, lens, 0.0, args.steps, args.warmup)
    res["d draw"] = forward_ms(dec, enc, formula, lens, TAU, args.steps, args.warmup)
    names = {"a": "fused getLoss, cross-entropy, eager", "b eager": "fused getLoss, SCST (tau = 1), eager",
             "b graph": "fused getLoss, SCST (tau = 1), CUDA graph",
             "c": "autograd route: rollout + dec(..., tau = 1) + torch PG loss + Adam",
             "d argmax": "no-grad decoder forward, p = 1, argmax (today's kernel)",
             "d draw": "no-grad decoder forward, p = 1, Gumbel draw (tau = 1)"}
    for k in ("a", "b eager", "b graph", "c", "d argmax", "d draw"):
        print("(%-8s) %-66s %8.2f ms" % (k, names[k], res[k]))
    Tn = formula.shape[1] - 1
    print("(b eager) / (a) = %.3f ; (c) / (b eager) = %.3f ; draw - argmax = %.2f us per step"
          % (res["b eager"] / res["a"], res["c"] / res["b eager"], (res["d draw"] - res["d argmax"]) * 1e3 / Tn))


if __name__ == "__main__":
    main()
