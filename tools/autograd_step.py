"""Train-step time at the cfg #2 workload (bf16, B=64, 128x512 images, T=150, V=500, dropout on) three ways:
  (a) the fused Img2SeqModel.getLoss, eager;
  (b) the fused getLoss replayed as a CUDA graph;
  (c) the reference's getLoss body (img2seq_torch.py:136-172) through autograd, with two torch.optim.Adam optimisers.
Times are CUDA-event means over the timed steps, after warm-up.  ``--profile`` prints the torch.profiler kernel table of one eager
step of (a) and one of (c).

  python tools/autograd_step.py [--steps 10] [--warmup 3] [--profile]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence

import bench_support as bs
from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel

B, H, W, T, V = 64, 128, 512, 150, 500


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False


def make_model(graph):
    torch.manual_seed(1234)
    cfg = Cfg()
    cfg.cuda_graph = graph
    m = Img2SeqModel(cfg, vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc")
    m.build_train()
    m.train_mode(True)
    return m


def reference_step(model, encoder_optimizer, decoder_optimizer, criterion, img, formula):
    """img2seq_torch.py:136-172; current torch's PackedSequence has four fields, hence ``.data``."""
    imgs = model.encoder(img)
    scores, caps_sorted, decode_lengths, alphas, sort_ind = model.decoder(imgs, formula, torch.LongTensor([[len(i)] for i in formula]))
    targets = caps_sorted[:, 1:]
    scores = pack_padded_sequence(scores, decode_lengths, batch_first=True).data
    targets = pack_padded_sequence(targets, decode_lengths, batch_first=True).data
    loss = criterion(scores, targets)
    alpha_c = 1.
    loss += alpha_c * ((1. - alphas.sum(dim=1)) ** 2).mean()
    decoder_optimizer.zero_grad()
    encoder_optimizer.zero_grad()
    loss.backward()
    decoder_optimizer.step()
    encoder_optimizer.step()
    return -loss.item()


def time_ms(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s (%s)" % (torch.cuda.get_device_name(), q.stdout.strip() or "power limit not reported"))
    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.cuda(), formula.cuda()
    steps = {}
    fused = make_model(False)
    steps["a"] = lambda: fused.getLoss(img, formula, None, None)
    graphed = make_model(True)
    steps["b"] = lambda: graphed.getLoss(img, formula, None, None)
    auto = make_model(False)
    opt_e = torch.optim.Adam(auto.encoder.parameters(), lr=1e-3)
    opt_d = torch.optim.Adam(auto.decoder.parameters(), lr=1e-3)
    crit = nn.CrossEntropyLoss()
    steps["c"] = lambda: reference_step(auto, opt_e, opt_d, crit, img, formula)
    names = {"a": "fused getLoss, eager", "b": "fused getLoss, CUDA graph", "c": "reference getLoss body, autograd + torch.optim.Adam"}
    res = {k: time_ms(f, args.steps, args.warmup) for k, f in steps.items()}
    for k in "abc":
        print("(%s) %-52s %8.2f ms/step" % (k, names[k], res[k]))
    print("(c) / (a) = %.3f" % (res["c"] / res["a"]))
    if args.profile:
        for k in "ac":
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                steps[k]()
                torch.cuda.synchronize()
            print("\n(%s) %s: kernel table of one step" % (k, names[k]))
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90))


if __name__ == "__main__":
    main()
