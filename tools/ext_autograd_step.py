"""Train-step time of the row-encoder extension at the cfg4 workload (``bench.py --workload cfg4`` shapes: bf16, B=64, 160x640
images, T=150, V=500, dropout on) three ways:
  (a) the fused Img2SeqRowModel.getLoss, eager;
  (b) the fused getLoss replayed as a CUDA graph;
  (c) through autograd: encoder -> row_encoder -> decoder2 -> the reference loss (img2seq_torch.py:147-159) -> loss.backward()
      -> one torch.optim.Adam over the four modules, returning -loss.item() like getLoss.
Times are CUDA-event means over the timed steps, after warm-up.  ``--profile`` prints the torch.profiler kernel table of one eager
step of (a) and one of (c) instead.

  python tools/ext_autograd_step.py [--steps 10] [--warmup 3] [--profile]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.nn.utils.rnn import pack_padded_sequence  # noqa: E402

import bench_support as bs  # noqa: E402
from latex_ocr_b200.data import SimpleVocab  # noqa: E402
from latex_ocr_b200.ext import Img2SeqRowModel  # noqa: E402

B, H, W, T, V = 64, 160, 640, 150, 500


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False


def make_model(graph):
    torch.manual_seed(1234)
    cfg = Cfg()
    cfg.cuda_graph = graph
    m = Img2SeqRowModel(cfg, vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc")
    m.build_train()
    m.train_mode(True)
    return m


def autograd_step(m, opt, img, formula, lengths):
    preds, caps, dl, alphas, _ = m.decoder2(m.row_encoder(m.encoder(img)), formula, lengths)
    scores = pack_padded_sequence(preds, dl, batch_first=True).data
    targets = pack_padded_sequence(caps[:, 1:], dl, batch_first=True).data
    loss = F.cross_entropy(scores, targets) + ((1. - alphas.sum(dim=1)) ** 2).mean()
    opt.zero_grad()
    loss.backward()
    opt.step()
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print("device: %s (%s)" % (torch.cuda.get_device_name(), q.stdout.strip() or "power limit / clocks not reported"))
    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.cuda(), formula.cuda()
    lengths = torch.full((B, 1), formula.shape[1], dtype=torch.long)      # every row at the padded length (img2seq_torch.py:144)
    names = {"a": "fused getLoss, eager", "b": "fused getLoss, CUDA graph",
             "c": "autograd: reference loss, backward(), torch.optim.Adam"}

    def make_step(k):
        """One model per way, built when it is timed (three cfg4 models at once need not fit next to other work)."""
        m = make_model(k == "b")
        if k != "c":
            return lambda: m.getLoss(img, formula)
        opt = torch.optim.Adam([p for mod in (m.encoder, m.row_encoder, m.decoder, m.layer2) for p in mod.parameters()], lr=1e-3)
        return lambda: autograd_step(m, opt, img, formula, lengths)

    if args.profile:
        for k in "ac":
            step = make_step(k)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                step()
                torch.cuda.synchronize()
            print("\n(%s) %s: kernel table of one step" % (k, names[k]))
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90))
            del step
            torch.cuda.empty_cache()
        return
    res = {}
    for k in "abc":
        step = make_step(k)
        res[k] = time_ms(step, args.steps, args.warmup)
        del step
        torch.cuda.empty_cache()
        print("(%s) %-55s %8.2f ms/step" % (k, names[k], res[k]), flush=True)
    print("(c) / (a) = %.3f   (c) / (b) = %.3f" % (res["c"] / res["a"], res["c"] / res["b"]))


if __name__ == "__main__":
    main()
