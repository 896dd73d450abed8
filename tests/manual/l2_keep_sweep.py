"""L2 residency of the decoder's attention rows (option att_l2_keep_mb), cfg #2 (bf16, B=64, 128x512 images, R=868, T=150).

att1 and encoder_out do not change inside a time loop; each attention launch streams 114 MB (forward) or 57 MB of enc (tensor-core
backward), more than the 50 MB L2.  The option keeps a fixed share of every launch's ring stages evict_last and streams the rest
evict_first.  In one run this prints the card, its power limit and max SM clock, then
  1. 200 back-to-back stand-alone forward (with mask bits) and backward launches per budget {0, 8, 16, 24, 32, 40} MiB: does a
     kept subset survive the streaming, and where is the knee of the usable L2;
  2. the same at B = 16 (28 MB of att1 + enc: fits the L2) with budget 0 and 40: the consumer-side ceiling at L2 speed;
  3. the graphed forward and backward time loops, µs per step, whole loop and attention only (dbg_skip), per budget.
Times are device events around the launches; the stand-alone launches use att_abi_pdl=1 like the time loop's.

    python tests/manual/l2_keep_sweep.py [--budgets 0,8,16,24,32,40] [--loop-budgets 0,16,24,32]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench_support as bs  # noqa: E402
from latex_ocr_b200 import _lib  # noqa: E402
from latex_ocr_b200.data import SimpleVocab  # noqa: E402
from latex_ocr_b200.img2seq import Img2SeqModel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--budgets", default="0,8,16,24,32,40")
ap.add_argument("--loop-budgets", default="0,16,24,32")
ap.add_argument("--launches", type=int, default=200)
args = ap.parse_args()
budgets = [int(v) for v in args.budgets.split(",")]
loop_budgets = [int(v) for v in args.loop_budgets.split(",")]

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("card:", q.stdout.strip() or torch.cuda.get_device_name(0), "| L2 %d MiB" % (torch.cuda.get_device_properties(0).L2_cache_size >> 20),
      "| library", os.environ.get("LO_LIB_DIR", "_C"), flush=True)

B, T, A, C = 64, 150, 512, 512


class Cfg:
    encoder_cnn = "vanilla"; positional_embeddings = True; lr_init = 1e-3; lr_method = "adam"; cuda_graph = False


m = Img2SeqModel(Cfg(), vocab=SimpleVocab(500), device="cuda:0", precision="bf16", impl="tc")
m.build_train(); m.train_mode(True)
img, formula = bs.synthetic_batch(B, 128, 512, 500, T, seed=1234)
img, formula = img.cuda(), formula.cuda()
for _ in range(2):
    m.train_step(img, formula)
torch.cuda.synchronize()
L = _lib.lib()
dec, enc = m.decoder, m.encoder
key = [k for k in dec._ws if k[0] == B and k[1] == T][0]
R = key[2]
t, a = dec._ws[key]["t"], dec._ws[key]["args"]
enc_out = enc._ws[(B, 128, 512)]["out"].view(B, R, C)
O1 = A + C + 4 * 512
st = _lib.stream_ptr()
dt = _lib.LO_BF16


def fwd(s, nb):
    o1 = t["out1"][s]
    _lib.check(L.lo_attention_forward_mask(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), O1, a.w_full,
                                           ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                           None, 0, None, _lib.ptr(t["att_mask"][s]), nb, R, A, C, _lib.ptr(t["work"]), st))


def bwd(s, nb):
    o1 = t["out1"][s]
    _lib.check(L.lo_attention_backward(_lib.ptr(t["att1"]), _lib.ptr(enc_out), dt, _lib.ptr(o1), ctypes.c_void_p(o1.data_ptr() + A * 4), O1,
                                       a.w_full, ctypes.c_void_p(t["alphas"].data_ptr() + s * R * 4), T * R, _lib.ptr(t["ctx"][s]),
                                       _lib.ptr(t["dxh"]), C + 512, _lib.ptr(t["dreg"]), R, ctypes.c_void_p(t["sreg"].data_ptr() + s * 4), T,
                                       ctypes.c_void_p(t["de"].data_ptr() + s * R * 4), _lib.ptr(t["dcat"][s]),
                                       ctypes.c_void_p(t["dcat"][s].data_ptr() + A * 4), O1, _lib.ptr(t["dctx"][s]), None,
                                       _lib.ptr(t["att_mask"][s]), nb, R, A, C, _lib.ptr(t["work"]), st))


def launches_us(fn, nb):
    def run():
        for i in range(args.launches):
            fn(i % T, nb)
    bs._time_ms(run, 1)                       # warm-up, then the timed window
    return bs._time_ms(run, 2) / args.launches * 1e3


def stand_alone(nb, budget):
    with _lib.option(att_abi_pdl=1, att_l2_keep_mb=budget):
        f, b = launches_us(fwd, nb), launches_us(bwd, nb)
    fb, bb = nb * R * (A + C) * 2 + nb * R * (4 + A // 8), nb * R * (C * 2 + A // 8 + 8)     # algorithmic bytes per launch
    r = {"B": nb, "keep_mb": budget, "fwd_us": round(f, 2), "fwd_TBps": round(fb / f / 1e6, 2), "bwd_us": round(b, 2),
         "bwd_TBps": round(bb / b / 1e6, 2)}
    print(json.dumps(r), flush=True)
    return r


def graph_ms(fn, iters=5):
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        fn(); fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            fn()
    torch.cuda.synchronize()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def loops(budget):
    def f():
        _lib.check(L.lo_decoder_forward(ctypes.byref(a), 1, _lib.stream_ptr()))

    def b():
        _lib.check(L.lo_decoder_backward(ctypes.byref(a), _lib.stream_ptr()))
    r = {"keep_mb": budget}
    with _lib.option(att_l2_keep_mb=budget):       # graphs capture the keep share with the launch arguments
        for mask, tag in ((8 | 1, "loop"), (8 | 1 | 4, "att_only")):
            with _lib.option(dbg_skip=mask):
                r["fwd_" + tag + "_us"] = round(graph_ms(f) / T * 1e3, 1)
                r["bwd_" + tag + "_us"] = round(graph_ms(b) / T * 1e3, 1)
    print(json.dumps(r), flush=True)


print("== stand-alone launches, %d back-to-back, B = %d" % (args.launches, B), flush=True)
for kb in budgets:
    stand_alone(B, kb)
print("== B = 16: att1 + enc = %.1f MB fit the L2" % (16 * R * (A + C) * 2 / 1e6), flush=True)
for kb in (0, 40):
    stand_alone(16, kb)
print("== graphed time loops (dbg_skip: 9 = loop, 13 = attention only), us per step", flush=True)
for kb in loop_budgets:
    loops(kb)
fwd(0, B); bwd(0, B); torch.cuda.synchronize()
