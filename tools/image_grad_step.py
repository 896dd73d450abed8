"""Cost of the image gradient at the cfg #2 workload (bf16, B=64, 128x512 images, T=150, V=500, dropout on):
  (a) conv1's data-gradient kernel alone (lo_conv1_pool_dgrad_code), bf16 and fp32 dpool: CUDA-event mean over --launches
      launches, and the bytes it must move (dpool + one code byte per pooled output and channel + the fp32 d image) over that time;
  (b) the reference's getLoss body through autograd with two torch.optim.Adam (tools/autograd_step.py), with and without
      img.requires_grad; the two arms alternate, --rounds times;
  (c) a saliency pass of a frozen model (every requires_grad False): encoder + decoder forward, the reference loss, backward to
      the image; no optimiser.
The card's name, power limit and max SM clock are printed with the numbers.

  python tools/image_grad_step.py [--steps 10] [--warmup 3] [--rounds 3] [--launches 200]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence

import bench_support as bs
from autograd_step import B, H, W, T, V, make_model, reference_step, time_ms
from latex_ocr_b200 import _lib


def device_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return "device: %s (%s)" % (torch.cuda.get_device_name(), q.stdout.strip() or "power limit / clock not reported")


def kernel_time(dtype, launches):
    """(a): µs per launch and GB/s over the bytes the kernel must move."""
    Hp, Wp = H // 2, W // 2
    g = torch.Generator().manual_seed(5)
    code = torch.randint(0, 8, (B, Hp, Wp, 64), generator=g, dtype=torch.uint8).cuda()
    dpool = torch.randn(B, Hp, Wp, 64, generator=g).to(dtype).cuda()
    w = torch.randn(64, 9, generator=g).cuda()
    dimg = torch.empty(B, H, W, device="cuda")
    L, dt = _lib.lib(), _lib.dt_of(dpool)
    args = (_lib.ptr(code), _lib.ptr(dpool), dt, _lib.ptr(w), 1.0, _lib.ptr(dimg), B, H, W, _lib.stream_ptr())
    for _ in range(10):
        _lib.check(L.lo_conv1_pool_dgrad_code(*args))
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(launches):
        L.lo_conv1_pool_dgrad_code(*args)
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / launches
    nbytes = dpool.numel() * (dpool.element_size() + 1) + dimg.numel() * 4
    return us, nbytes


def saliency_step(model, crit, img, formula):
    """(c): frozen model, gradient of the reference loss w.r.t. the image only."""
    x = img.detach().requires_grad_(True)
    scores, caps, dl, alphas, _ = model.decoder(model.encoder(x), formula, torch.LongTensor([[len(i)] for i in formula]))
    loss = crit(pack_padded_sequence(scores, dl, batch_first=True).data,
                pack_padded_sequence(caps[:, 1:], dl, batch_first=True).data)
    loss = loss + ((1. - alphas.sum(dim=1)) ** 2).mean()
    loss.backward()
    return x.grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    print(device_line())
    for dtype in (torch.bfloat16, torch.float32):
        us, nbytes = kernel_time(dtype, args.launches)
        print("(a) conv1 dgrad kernel, %-8s dpool: %8.1f us/launch, %6.1f MB -> %7.1f GB/s (%.0f%% of the 3.35 TB/s data-sheet HBM3)"
              % (str(dtype).split(".")[1], us, nbytes / 1e6, nbytes / us / 1e3, 100 * nbytes / us / 1e3 / 3350))
    img, formula = bs.synthetic_batch(B, H, W, V, T, seed=1234)
    img, formula = img.float().cuda(), formula.cuda()
    auto = make_model(False)
    opt_e = torch.optim.Adam(auto.encoder.parameters(), lr=1e-3)
    opt_d = torch.optim.Adam(auto.decoder.parameters(), lr=1e-3)
    crit = nn.CrossEntropyLoss()
    img_grad = img.clone().requires_grad_(True)
    arms = {"without": lambda: reference_step(auto, opt_e, opt_d, crit, img, formula),
            "with": lambda: reference_step(auto, opt_e, opt_d, crit, img_grad, formula)}
    res = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, f in arms.items():
            res[k].append(time_ms(f, args.steps, args.warmup))
    for k in arms:
        print("(b) autograd step %-7s img.requires_grad: %s ms/step" % (k, " ".join("%.2f" % t for t in res[k])))
    print("(b) with / without (means): %.4f" % (sum(res["with"]) / sum(res["without"])))
    frozen = make_model(False)
    for p in list(frozen.encoder.parameters()) + list(frozen.decoder.parameters()):
        p.requires_grad_(False)
    sal = [time_ms(lambda: saliency_step(frozen, crit, img, formula), args.steps, args.warmup) for _ in range(args.rounds)]
    print("(c) saliency pass, frozen model (forward + backward to the image): %s ms" % " ".join("%.2f" % t for t in sal))


if __name__ == "__main__":
    main()
