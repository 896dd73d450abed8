"""Decode of the row-encoder extension (ext.greedy_decode / ext.beam_decode) at cfg #4 shapes: 256 images of 160 x 640 px
(R = 18 x 78 = 1404 regions), V = 500, bf16 storage on the wgmma / mma.sync kernels, random-init weights.

  1. per step, on one encoder_out: the two-layer time loop (lo_decoder2_greedy / lo_decoder2_beam) against the one-layer loop
     (lo_decoder_greedy_hist / lo_decoder_beam_div) on the same argument block, greedy (256 rows) and beam 5 (1280 rows).  The
     library runs max_length_formula + 2 = 152 steps whatever the tokens, so ms / step = loop time / 152; the difference of the
     two is what layer 2 (two skinny GEMMs and one cell launch per step, two gathers per beam step) adds.
  2. end to end: ext.greedy_decode / ext.beam_decode on host images (CNN + row encoder + loop + trimming), generated tokens / s =
     rows x 152 / time.
  3. a cfg #5-style list: 256 images of height 160 and widths 64..1024, every image at its own size in one time loop.
Times are the faster of two CUDA-synchronised passes after one warm-up pass; the card's name, power limit and SM clock are printed.

    python tools/ext_decode_bench.py        (one JSON line on stdout)
"""
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from latex_ocr_b200 import _lib, decode, ext
from latex_ocr_b200._lib import stream_ptr
from latex_ocr_b200.ext import Img2SeqRowModel

V, N_IMG, H, W, MAX_LEN, BEAM = 500, 256, 160, 640, 150, 5
STEPS = MAX_LEN + 2
START, END = V - 2, V - 1


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"


def timed(fn):
    best = None
    for rep in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if rep and (best is None or dt < best):
            best = dt
    return best


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                      # the numbers stay valid, only the label is missing
        return "nvidia-smi failed: %s" % e


def loops(m, img, rows_per_img):
    """(one-layer, two-layer) loop seconds on one prepared argument block"""
    L = _lib.lib()
    a, ws, N, _ = decode._prepare(m, img, rows_per_img, STEPS, m.row_encoder.forward_raw)
    B = N * rows_per_img
    dev = m.device
    l2 = m.layer2.decode_layer(a)
    if rows_per_img == 1:
        tok = torch.zeros(B, STEPS, dtype=torch.int64, device=dev)
        fin = torch.zeros(B, dtype=torch.int32, device=dev)
        hist = torch.zeros(B, STEPS, dtype=torch.int32, device=dev)
        rest = (START, END, STEPS, tok.data_ptr(), fin.data_ptr(), hist.data_ptr(), stream_ptr())
        one = lambda: _lib.check(L.lo_decoder_greedy_hist(ctypes.byref(a), *rest))
        two = lambda: _lib.check(L.lo_decoder2_greedy(ctypes.byref(a), ctypes.byref(l2), *rest))
    else:
        ids = torch.zeros(N, STEPS, rows_per_img, dtype=torch.int64, device=dev)
        par = torch.zeros_like(ids)
        hist = torch.zeros(N, STEPS, rows_per_img, dtype=torch.int32, device=dev)
        logp = torch.zeros(N, rows_per_img, device=dev)
        rest = (START, END, STEPS, ids.data_ptr(), par.data_ptr(), hist.data_ptr(), logp.data_ptr(), 1.0, 0.0, None, None)
        one = lambda: _lib.check(L.lo_decoder_beam_div(ctypes.byref(a), *rest, stream_ptr()))
        two = lambda: _lib.check(L.lo_decoder2_beam(ctypes.byref(a), ctypes.byref(l2), *rest, None, stream_ptr()))
    t1, t2 = timed(one), timed(two)
    return {"rows": B, "R": a.R, "one_layer_ms_per_step": 1e3 * t1 / STEPS, "two_layer_ms_per_step": 1e3 * t2 / STEPS,
            "layer2_ms_per_step": 1e3 * (t2 - t1) / STEPS, "two_layer_loop_tokens_per_s": B * STEPS / t2}


def main():
    torch.manual_seed(0)
    m = Img2SeqRowModel(Cfg(), n_tok=V, device="cuda", precision="bf16", impl="tc")
    m.build_train()
    m.train_mode(False)
    g = torch.Generator().manual_seed(5)
    img = torch.where(torch.rand(N_IMG, 1, H, W, generator=g) < 0.1, torch.randint(0, 255, (N_IMG, 1, H, W), generator=g),
                      torch.full((N_IMG, 1, H, W), 255)).to(torch.uint8)
    out = {"card": card(), "workload": "cfg4 %d x %dx%d, V=%d, bf16 tc, %d steps" % (N_IMG, H, W, V, STEPS)}
    with torch.no_grad():
        out["greedy_loop"] = loops(m, img, 1)
        out["beam5_loop"] = loops(m, img, BEAM)
    t = timed(lambda: ext.greedy_decode(m, img, START, END, MAX_LEN))
    out["greedy_end_to_end"] = {"s": t, "tokens_per_s": N_IMG * STEPS / t, "images_per_s": N_IMG / t}
    t = timed(lambda: ext.beam_decode(m, img, START, END, BEAM, max_length_formula=MAX_LEN))
    out["beam5_end_to_end"] = {"s": t, "tokens_per_s": N_IMG * BEAM * STEPS / t, "images_per_s": N_IMG / t}
    widths = [64 * (1 + (i * 7) % 16) for i in range(N_IMG)]             # 64..1024 px, 16 widths
    imgs = [torch.where(torch.rand(1, H, w, generator=g) < 0.1, torch.randint(0, 255, (1, H, w), generator=g),
                        torch.full((1, H, w), 255)).to(torch.uint8) for w in widths]
    t = timed(lambda: ext.greedy_decode(m, imgs, START, END, MAX_LEN))
    out["mixed_widths_greedy"] = {"s": t, "tokens_per_s": N_IMG * STEPS / t, "images_per_s": N_IMG / t}
    t = timed(lambda: ext.beam_decode(m, imgs, START, END, BEAM, max_length_formula=MAX_LEN))
    out["mixed_widths_beam5"] = {"s": t, "tokens_per_s": N_IMG * BEAM * STEPS / t, "images_per_s": N_IMG / t}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
