"""Cost of the length and coverage penalties of beam search (lo_beam_penalty) on cfg #5 (BASELINE.json configs[4]): the ragged beam-5
decode of tools/ragged_decode_bench.py (256 images of height 64, widths 64..1024, bf16 storage on the wgmma / mma.sync kernels, one
Img2SeqModel.predict_images call, host uint8 images in, token ids out, 152 steps: random-init weights never emit END) without
penalties and with (length_penalty, coverage_penalty) = (0.6, 0.2).  The two arms alternate inside one process, three timed passes
each after a warm-up pass of each, and the faster pass of each arm is reported as tokens/s.

A separate torch.profiler run of the penalised arm gives the per-step device time of the coverage kernel, the beam step kernel and
the ragged attention kernel, and the coverage kernel's bytes per step (attention rows read, coverage read by parent and written:
3 x 4 bytes per region of every row) against the attention launch's (enc and att1 rows in bf16 once per image, the attention rows
written).  The card's name, power limit and maximum SM clock are printed beside the numbers.

    python tools/beam_penalty_bench.py [--out DIR]     (one JSON line on stdout; the profiler table under DIR if given)
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from latex_ocr_b200.data import SimpleVocab
from latex_ocr_b200.img2seq import Img2SeqModel

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ragged_decode_bench as rdb          # noqa: E402  (the cfg #5 workload and the card query)

BEAM = 5
ARMS = {"no_penalty": (0.0, 0.0), "penalty_0.6_0.2": (0.6, 0.2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure on the CPU")
    m = Img2SeqModel(rdb.Cfg(), vocab=SimpleVocab(rdb.V), device="cuda:0", precision="bf16", impl="tc").build_pred()
    m.train_mode(False)
    cfg = m._config
    cfg.max_length_formula = rdb.MAX_LEN
    cfg.decoding, cfg.beam_size = "beam_search", BEAM
    imgs, _ = rdb.workload()

    def run(arm):
        cfg.length_penalty, cfg.coverage_penalty = ARMS[arm]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ids = m.predict_images(imgs)[0]
        torch.cuda.synchronize()
        return time.perf_counter() - t0, sum(len(s.split()) if isinstance(s, str) else len(s) for s in ids)

    out = {"card": rdb.card(), "workload": "cfg5 ragged beam %d: %d images %d x {%s} px, bf16 + tc, %d decode steps; arms alternate, "
                                           "fastest of 3 timed passes after a warm-up pass" % (BEAM, rdb.N_IMG, rdb.HEIGHT,
                                                                                            ",".join(map(str, rdb.WIDTHS)),
                                                                                            rdb.MAX_LEN + 2)}
    best = {}
    for rep in range(4):
        for arm in ARMS:
            dt, toks = run(arm)
            if rep > 0 and (arm not in best or dt < best[arm][0]):
                best[arm] = (dt, toks)
    for arm, (dt, toks) in best.items():
        out["%s_tok_s" % arm] = toks / dt
        out["%s_seconds" % arm] = dt
    out["penalty_time_ratio"] = best["penalty_0.6_0.2"][0] / best["no_penalty"][0]

    from torch.profiler import ProfilerActivity, profile
    cfg.length_penalty, cfg.coverage_penalty = ARMS["penalty_0.6_0.2"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.predict_images(imgs)
        torch.cuda.synchronize()
    steps = rdb.MAX_LEN + 2
    for key, name in (("beam_coverage_kernel", "coverage"), ("beam_step_kernel", "beam_step"), ("attention_fwd_ragged_kernel", "attention")):
        ev = [e for e in prof.key_averages() if key in e.key]
        if not ev:
            raise SystemExit("profile has no %s" % key)
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in ev)
        out["%s_launches" % name] = sum(e.count for e in ev)
        out["%s_us_per_step" % name] = us / steps
    counts = []
    for x in imgs:
        h, w = m.encoder.out_hw(x.shape[0], x.shape[1])
        counts.append(h * w)
    A = C = 512
    out["coverage_bytes_per_step"] = sum(BEAM * r * 12 + BEAM * 12 for r in counts)   # alpha + cov in + cov out; finished, parent, term
    out["attention_bytes_per_step"] = sum(r * (A + C) * 2 + BEAM * r * 4 for r in counts)
    out["coverage_GB_s"] = out["coverage_bytes_per_step"] / (out["coverage_us_per_step"] * 1e-6) / 1e9
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "beam_penalty_profile.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=25))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
