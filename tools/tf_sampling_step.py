"""Cost of scheduled sampling and self-critical training on the TensorFlow-flavour model at the cfg #2 workload (bf16, B=64,
128x512 images, T=150, V=500, the TF dims of configs/model.json, dropout off, tau = 1):
  (a) the fused cross-entropy step, img2seq_tf.Img2SeqModel.train_step;
  (b) the same step with set_sampling_prob(0.25);
  (c) the same step with set_self_critical(1.0) (sample pass, greedy rollout, reward, policy gradient, generic backward);
  (d) the autograd route of SCST: encoder, greedy decode under no_grad, Decoder.train_outputs(..., sampling_prob=1,
      sampling_temperature=1), scst.rewards(layout="tf"), the policy-gradient loss in plain torch, backward, torch.optim.Adam;
  (e) the in-loop head: a no-grad Decoder.train_outputs at p = 1 with coins that never sample (the per-step head GEMM and the
      sampling pointwise kernel) against the teacher-forced one (the hoisted head GEMM); the difference over T is the cost per step.
Times are CUDA-event means over the timed steps after warm-up.  The card's name, power limit and max SM clock are printed with
the numbers.

  python tools/tf_sampling_step.py [--steps 10] [--warmup 3]
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

import bench_support as bs  # noqa: E402
from attention_autograd_step import device_line  # noqa: E402
from latex_ocr_b200 import scst  # noqa: E402
from tf_autograd_step import B, H, T, V, W, make_model, time_ms  # noqa: E402

TAU = 1.0


def autograd_scst_step(model, opt, img, formula, end_id):
    """(d): the SCST recipe of INTEGRATION.md (TF section) through autograd."""
    dec = model.decoder
    N, Tn = formula.shape
    enc = model.encoder(img)
    with torch.no_grad():
        greedy = dec.decode(enc.detach(), max_steps=Tn).ids
    logits, _ = dec.train_outputs(enc, formula, sampling_prob=1.0, sampling_temperature=TAU)
    fed = dec.last_fed_tokens
    _, _, adv, n_len = scst.rewards(fed, formula, end_id, greedy=greedy, layout="tf")
    lp = torch.log_softmax(logits / TAU, dim=-1).gather(2, fed[:, :, None])[:, :, 0]
    steps = torch.arange(Tn, device=lp.device)[None, :] < n_len[:, None]
    loss = -(adv[:, None] * lp * steps).sum() / N
    opt.zero_grad()
    loss.backward()
    opt.step()
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print(device_line())
    img, formula = bs.synthetic_batch(B, H, W, V, T - 1, seed=1234)       # T columns: tokens, END, PAD
    img, formula = img.to(torch.uint8).cuda(), formula.cuda()
    lengths = (formula != V - 2).sum(dim=1).to(torch.int32)
    f_host, l_host = formula.cpu(), lengths.cpu()
    res = {}
    m = make_model()
    step = lambda: m.train_step(img, (f_host, l_host))
    res["a"] = time_ms(step, args.steps, args.warmup)
    m.set_sampling_prob(0.25)
    res["b"] = time_ms(step, args.steps, args.warmup)
    m.set_sampling_prob(0.0)
    m.set_self_critical(TAU)
    res["c"] = time_ms(step, args.steps, args.warmup)
    print("fused SCST stats [L, mean r_sample, mean r_greedy, mean n_b]:", [round(x, 4) for x in step().tolist()])
    m.set_self_critical(None)
    auto = make_model()
    opt = torch.optim.Adam(list(auto.encoder.parameters()) + list(auto.decoder.parameters()), lr=1e-3)
    res["d"] = time_ms(lambda: autograd_scst_step(auto, opt, img, formula, V - 1), args.steps, args.warmup)
    dec = m.decoder
    with torch.no_grad():
        enc = m.encoder(img)

    def forward(p):
        with torch.no_grad():
            dec.train_outputs(enc, formula, sampling_prob=p)

    res["e tf"] = time_ms(lambda: forward(0.0), args.steps, args.warmup)
    dec._ss_u = torch.ones(B, T, device="cuda")                         # coins of 1: nothing is sampled, the loop is the same
    res["e head"] = time_ms(lambda: forward(1.0), args.steps, args.warmup)
    dec._ss_u = None
    names = {"a": "fused train_step, cross-entropy", "b": "fused train_step, set_sampling_prob(0.25)",
             "c": "fused train_step, set_self_critical(1.0)",
             "d": "autograd SCST: rollout + train_outputs(tau = 1) + torch PG loss + Adam",
             "e tf": "no-grad train_outputs, teacher forcing (hoisted head)",
             "e head": "no-grad train_outputs, p = 1, u = 1 (in-loop head)"}
    for k in ("a", "b", "c", "d", "e tf", "e head"):
        print("(%-6s) %-72s %8.2f ms" % (k, names[k], res[k]))
    print("(b) / (a) = %.3f ; (c) / (a) = %.3f ; (d) / (c) = %.3f ; in-loop head: %+.2f us per step"
          % (res["b"] / res["a"], res["c"] / res["a"], res["d"] / res["c"], (res["e head"] - res["e tf"]) * 1e3 / T))


if __name__ == "__main__":
    main()
