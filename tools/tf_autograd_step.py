"""TensorFlow-flavour train-step time at the cfg #2 workload (bf16, B=64, 128x512 images, T=150, V=500, the TF dims of
configs/model.json: num_units 512, dim_e 256, dim_o 512, dim_embeddings 80, dropout off) two ways:
  (a) the fused step, img2seq_tf.Img2SeqModel.train_step (masked CE and its backward in the kernels, fused TF Adam);
  (b) through autograd: EncoderCNN(input_norm="tf") -> Decoder.train_outputs -> masked CE in torch -> loss.backward() ->
      torch.optim.Adam over both modules.
Times are CUDA-event means over the timed steps, after warm-up.  ``--profile`` prints the torch.profiler kernel table of one
step of each instead.

  python tools/tf_autograd_step.py [--steps 10] [--warmup 3] [--profile]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench_support as bs  # noqa: E402
from latex_ocr_b200.data import SimpleVocab  # noqa: E402
from latex_ocr_b200.img2seq_tf import Img2SeqModel  # noqa: E402

B, H, W, T, V = 64, 128, 512, 150, 500


class Cfg:
    attn_cell_config = {"num_units": 512, "dim_e": 256, "dim_o": 512, "dim_embeddings": 80}
    max_length_formula = 150; decoding = "greedy"; lr_init = 1e-3; lr_method = "adam"; clip = -1; dropout = 1.0


def make_model():
    torch.manual_seed(1234)
    return Img2SeqModel(Cfg(), vocab=SimpleVocab(V), device="cuda", precision="bf16", impl="tc").build_train()


def masked_ce(logits, formula, lengths):
    """img2seq.py:68-71: mean sparse softmax CE over sequence_mask(lengths)."""
    mask = torch.arange(logits.shape[1], device=logits.device)[None, :] < lengths[:, None]
    return torch.nn.functional.cross_entropy(logits[mask], formula[mask])


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
    img, formula = bs.synthetic_batch(B, H, W, V, T - 1, seed=1234)       # T columns: tokens, END, PAD
    img, formula = img.to(torch.uint8).cuda(), formula.cuda()
    lengths = (formula != V - 2).sum(dim=1).to(torch.int32)               # tokens incl. END
    steps = {}
    fused = make_model()
    f_host, l_host = formula.cpu(), lengths.cpu()
    steps["a"] = lambda: fused.train_step(img, (f_host, l_host))
    auto = make_model()
    opt = torch.optim.Adam(list(auto.encoder.parameters()) + list(auto.decoder.parameters()), lr=1e-3)

    def autograd_step():
        opt.zero_grad()
        logits, _ = auto.decoder.train_outputs(auto.encoder(img), formula)
        loss = masked_ce(logits, formula, lengths)
        loss.backward()
        opt.step()
        return loss

    steps["b"] = autograd_step
    names = {"a": "fused Img2SeqModel.train_step (TF Adam)", "b": "autograd: masked CE, backward(), torch.optim.Adam"}
    if args.profile:
        for k in "ab":
            for _ in range(args.warmup):
                steps[k]()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                steps[k]()
                torch.cuda.synchronize()
            print("\n(%s) %s: kernel table of one step" % (k, names[k]))
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90))
        return
    res = {k: time_ms(f, args.steps, args.warmup) for k, f in steps.items()}
    for k in "ab":
        print("(%s) %-52s %8.2f ms/step" % (k, names[k], res[k]))
    print("(b) / (a) = %.3f" % (res["b"] / res["a"]))


if __name__ == "__main__":
    main()
