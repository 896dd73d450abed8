"""Sampling decode (decode.sample_decode, lo_decoder_sample) next to greedy and beam search on cfg #5 (BASELINE.json configs[4]):
the 256 images of tools/ragged_decode_bench.py (height 64, widths 64..1024, host uint8 images in one list), bf16 storage on the
wgmma / mma.sync kernels, 152 steps (random-init weights never emit END).  Arms: greedy, beam 8 and sample 8 (tau 1, top-k 0,
top-p 0.9: the filtered path with the shared-memory sort).  The arms alternate inside one process, three timed passes each after a
warm-up pass of each; each pass is timed with CUDA events around the call and the fastest pass is reported as generated tokens/s
(rows x steps: one token per image for greedy, eight for beam and sample).

A separate torch.profiler run of the sample arm gives the per-step device time of sample_step_kernel and of the ragged attention
kernel, and the sample kernel's bytes per step (one fp32 logits row per row) against its time.  The card's name, power limit and
maximum SM clock, read in the same process, are printed beside the numbers.

    python tools/sample_decode_bench.py [--out DIR]     (one JSON line on stdout; the profiler table under DIR if given)
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from latex_ocr_b200 import decode
from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ragged_decode_bench as rdb          # noqa: E402  (the cfg #5 workload and the card query)

N_S = 8
START, END = rdb.V - 2, rdb.V - 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    m = Img2SeqModel(rdb.Cfg(), vocab=SimpleVocab(rdb.V), device="cuda:0", precision="bf16", impl="tc").build_pred()
    m.train_mode(False)
    imgs, _ = rdb.workload()
    arms = {
        "greedy": (1, lambda: decode.greedy_decode(m, imgs, START, END, rdb.MAX_LEN)),
        "beam8": (N_S, lambda: decode.beam_decode(m, imgs, START, END, N_S, rdb.MAX_LEN)[0]),
        "sample8": (N_S, lambda: decode.sample_decode(m, imgs, START, END, N_S, 1.0, 0, 0.9, rdb.MAX_LEN, seed=1)[0]),
    }

    def run(arm):
        rows, fn = arms[arm]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        ids = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3, len(imgs) * rows * ids.shape[-1]

    out = {"card": rdb.card(), "workload": "cfg5: %d images %d x {%s} px in one list, bf16 + tc, %d decode steps; greedy, beam %d, "
                                           "sample %d (tau 1, top-p 0.9); arms alternate, fastest of 3 timed passes after a warm-up "
                                           "pass, CUDA events" % (rdb.N_IMG, rdb.HEIGHT, ",".join(map(str, rdb.WIDTHS)),
                                                                  rdb.MAX_LEN + 2, N_S, N_S)}
    best = {}
    for rep in range(4):
        for arm in arms:
            dt, toks = run(arm)
            if rep > 0 and (arm not in best or dt < best[arm][0]):
                best[arm] = (dt, toks)
    for arm, (dt, toks) in best.items():
        out["%s_tok_s" % arm] = toks / dt
        out["%s_seconds" % arm] = dt

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arms["sample8"][1]()
        torch.cuda.synchronize()
    steps = rdb.MAX_LEN + 2
    for key, name in (("sample_step_kernel", "sample"), ("attention_fwd_ragged_kernel", "attention")):
        ev = [e for e in prof.key_averages() if key in e.key]
        if not ev:
            raise SystemExit("profile has no %s" % key)
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
        out["%s_launches" % name] = sum(e.count for e in ev)
        out["%s_us_per_step" % name] = us / steps
    out["sample_bytes_per_step"] = len(imgs) * N_S * rdb.V * 4
    out["sample_GB_s"] = out["sample_bytes_per_step"] / (out["sample_us_per_step"] * 1e-6) / 1e9
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sample_decode_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=25))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
